"""Per-phase time breakdown of the persistent decode kernel from its %globaltimer trace (run on the GPU box)."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gguf_synth as S  # noqa: E402


def main():
    os.environ["GL_MEGA_TRACE"] = "1"
    os.environ.setdefault("GL_PREFILL", "1")
    from gridllm_b200 import native as N
    path = "/dev/shm/prof_llama3_8b.gguf"
    if not os.path.exists(path):
        S.build_model(path, S.LLAMA3_8B, "q4_k_m", seed=1234, mode="random", with_vocab=False)
    e = N.Engine(path, max_ctx=1024)
    ctx = int(sys.argv[1]) if len(sys.argv) > 1 else 576
    ms, _ = e.time_decode(ctx, 8)
    lib = N.load_library()
    cap = 132 * 200 * 4
    buf = np.zeros(cap, dtype=np.uint64)
    nc, nph = C.c_int32(), C.c_int32()
    rc = lib.gl_debug_mega_trace(e._h, buf.ctypes.data_as(C.c_void_p), cap, C.byref(nc), C.byref(nph))
    assert rc == 0, lib.gl_last_error()
    t = buf[: nc.value * (nph.value + 1) * 4].reshape(nc.value, nph.value + 1, 4)[:, : nph.value, :].astype(np.int64)
    names = ["QKV", "ATTN", "O", "GATEUP", "DOWN"]
    print(f"ctx {ctx}: {ms:.3f} ms/token; phases {nph.value}; ns per phase, mean over CTAs (max over CTAs)")
    print(f"{'phase':8s} {'prologue':>16s} {'work':>16s} {'barrier':>16s} {'total':>10s}")
    tot = {}
    for ph in range(nph.value):
        kind = names[ph % 5] if ph < nph.value - 1 else "HEAD"
        pro = t[:, ph, 1] - t[:, ph, 0] if kind != "ATTN" else np.zeros(nc.value, np.int64)
        work = t[:, ph, 2] - np.where(kind != "ATTN", t[:, ph, 1], t[:, ph, 0])
        bar = t[:, ph, 3] - t[:, ph, 2]
        whole = (t[:, ph, 3] - t[:, ph, 0]).mean()
        d = tot.setdefault(kind, [[], [], [], []])
        d[0].append((pro.mean(), pro.max())); d[1].append((work.mean(), work.max())); d[2].append((bar.mean(), bar.max())); d[3].append(whole)
    grand = 0.0
    for k in names + ["HEAD"]:
        d = tot[k]
        f = lambda a: f"{np.mean([x[0] for x in a]):7.0f} ({np.mean([x[1] for x in a]):6.0f})"
        w = float(np.mean(d[3])) * len(d[3])
        grand += w
        print(f"{k:8s} {f(d[0]):>16s} {f(d[1]):>16s} {f(d[2]):>16s} {np.mean(d[3]):10.0f}   x{len(d[3])} = {w / 1e3:8.1f} us")
    print(f"sum of phases {grand / 1e6:.3f} ms")
    # busiest / idlest CTA in the gate/up phase of a middle layer
    ph = 5 * 16 + 3
    w = t[:, ph, 2] - t[:, ph, 1]
    print("GATEUP layer 16 work ns: min %d median %d max %d" % (w.min(), np.median(w), w.max()))
    e.close()


if __name__ == "__main__":
    main()
