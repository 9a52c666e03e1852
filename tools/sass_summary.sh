#!/bin/bash
# Hopper-native evidence that can be checked from the tree: per kernel of the shipped library, how many of the SASS
# instructions of the sm_90a paths -- HGMMA (wgmma), UTMALDG (2-D TMA), UBLKCP (1-D bulk copy), SYNCS (mbarrier),
# IDP.4A (dp4a), HMMA (mma.sync) -- appear.
# Usage: tools/sass_summary.sh [lib.so]        (cuobjdump needs no GPU)
LIB="${1:-gridllm_b200/libgridllm_native.so}"
echo "# SASS summary of $LIB ($(date -u +%Y-%m-%dT%H:%MZ)), cuobjdump $(cuobjdump --version | tail -1)"
echo "# kernel | HGMMA UTMALDG UBLKCP SYNCS IDP.4A HMMA | instructions"
cuobjdump -sass "$LIB" | awk '
/Function :/ { if (name != "") emit(); name=$3; delete c; n=0; next }
/^[ \t]+\/\*[0-9a-f]+\*\// { n++; op=$2; sub(/;.*/, "", op);
    if (op ~ /^HGMMA/) c["HGMMA"]++; if (op ~ /^UTMALDG/) c["UTMALDG"]++; if (op ~ /^UBLKCP/) c["UBLKCP"]++;
    if (op ~ /^SYNCS/) c["SYNCS"]++; if (op ~ /^IDP\.4A/) c["IDP.4A"]++; if (op ~ /^HMMA/) c["HMMA"]++ }
function emit() { printf "%s | %d %d %d %d %d %d | %d\n", name, c["HGMMA"], c["UTMALDG"], c["UBLKCP"], c["SYNCS"], c["IDP.4A"], c["HMMA"], n }
END { if (name != "") emit() }' | while IFS= read -r line; do
    k="${line%% |*}"; rest="${line#* |}"
    echo "$(echo "$k" | c++filt | sed 's/gl::(anonymous namespace):://; s/(.*//') |$rest"
done | sort
