"""Device-side timeline of one decode step of the per-op CUDA-graph path (GL_TRACE=1): for every GEMV / attention launch,
%globaltimer at kernel entry, after griddepcontrol.wait, after the prologue and at the end, for the first and last CTA."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import gguf_synth as S  # noqa: E402


def main():
    os.environ["GL_TRACE"] = "1"
    os.environ.setdefault("GL_PREFILL", "1")
    from gridllm_b200 import native as N
    path = "/dev/shm/prof_llama3_8b.gguf"
    if not os.path.exists(path):
        S.build_model(path, S.LLAMA3_8B, "q4_k_m", seed=1234, mode="random", with_vocab=False)
    e = N.Engine(path, max_ctx=1024)
    ctx = int(sys.argv[1]) if len(sys.argv) > 1 else 576
    ms, nl = e.time_decode(ctx, 8)
    lib = N.load_library()
    cap = 512 * 16
    buf = np.zeros(cap, dtype=np.uint64)
    n = C.c_int32()
    lib.gl_debug_perop_trace.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
    rc = lib.gl_debug_perop_trace(e._h, buf.ctypes.data_as(C.c_void_p), cap, C.byref(n))
    assert rc == 0, lib.gl_last_error()
    t8 = buf.reshape(512, 2, 8).astype(np.int64)
    t = t8[:, :, :4]
    # launch order of a step: embed, 32 x (QKV, attn, O, gate/up, down), lm_head, sampler; only GEMV / attention launches stamp
    names = ["QKV", "ATTN", "O", "GATEUP", "DOWN"]
    rows = []
    for il in range(32):
        for k in range(5):
            rows.append((f"{names[k]}", t[1 + 5 * il + k]))
    rows.append(("HEAD", t[1 + 160]))
    print(f"ctx {ctx}: {ms:.4f} ms/token, {nl} launches; ns, first CTA | last CTA; gap = entry - previous kernel's end (max of both CTAs)")
    print(f"{'kernel':8s} {'gap':>7s} {'wait':>7s} {'prolog':>7s} {'work':>7s} {'total':>7s} | {'wait':>7s} {'prolog':>7s} {'work':>7s}")
    agg = {}
    prev_end = None
    t_first = None
    for name, r in rows:
        a, b = r[0], r[1]
        if a[0] == 0:
            continue
        if t_first is None:
            t_first = a[0]
        end = max(a[3], b[3])
        gap = (min(a[0], b[0]) - prev_end) if prev_end is not None else 0
        d = agg.setdefault(name, [])
        d.append((gap, a[1] - a[0], a[2] - a[1], a[3] - a[2], end - min(a[0], b[0]), b[1] - b[0], b[2] - b[1], b[3] - b[2]))
        prev_end = end
    for name in names + ["HEAD"]:
        d = np.array(agg[name], dtype=np.float64)
        m = d.mean(axis=0)
        print(f"{name:8s} {m[0]:7.0f} {m[1]:7.0f} {m[2]:7.0f} {m[3]:7.0f} {m[4]:7.0f} | {m[5]:7.0f} {m[6]:7.0f} {m[7]:7.0f}   x{len(d)}")
    print(f"span first QKV entry -> lm_head end: {(prev_end - t_first) / 1e3:.1f} us")
    # prologue split (GEMV launches): wait-done -> x arrived -> snap done -> planes ready (named barrier)
    print('prologue split, first CTA, mean ns: x arrives | snap | barrier')
    for k, name in enumerate(names):
        if name == 'ATTN':
            continue
        r = np.array([t8[1 + 5 * il + k][0] for il in range(32)], dtype=np.float64)
        print(f'{name:8s} {np.mean(r[:, 4] - r[:, 1]):7.0f} {np.mean(r[:, 5] - r[:, 4]):7.0f} {np.mean(r[:, 2] - r[:, 5]):7.0f}')
    r = np.array([t8[1 + 5 * il + 1][0] for il in range(32)], dtype=np.float64)
    o = np.array([t8[1 + 5 * il + 2][0] for il in range(32)], dtype=np.float64)
    print('ATTN tail, mean ns after the upstream wait (first CTA): pages done %.0f | merged %.0f | attn_output wait over %.0f'
          % (np.mean(r[:, 2] - r[:, 1]), np.mean(r[:, 3] - r[:, 1]), np.mean(o[:, 1] - r[:, 1])))
    # one layer in detail
    il = 16
    base = None
    for k in range(5):
        r = t[1 + 5 * il + k]
        if base is None:
            base = r[0][0]
        print(f"layer {il} {names[k]:7s} first CTA {[int(x - base) for x in r[0]]}  last CTA {[int(x - base) for x in r[1]]}")
    e.close()


if __name__ == "__main__":
    main()
