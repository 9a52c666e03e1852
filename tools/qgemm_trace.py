"""Device timeline of the quantised GEMMs inside one REPLAYED batched step (run on an H100 with GL_QGEMM_TRACE=1).

The kernel stamps %globaltimer per CTA at: 0 entry, 1 prologue done, 2 first weight copy issued, 3 first qtile landed,
4 unpack warps done (5 is not written), 6 last accumulator complete, 7 epilogue done, 8 upstream kernel complete
(griddepcontrol.wait returned), 9 last MMA complete.  A captured graph keeps the trace slot of its capture, so after the replays the buffer holds
the stamps of the LAST replay of every launch.  usage: qgemm_trace.py <batch> <ctx>"""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["GL_QGEMM_TRACE"] = "1"

SLOTS, GRID = 10, 132
NAMES = ["entry", "prologue", "tma0", "qtile0", "unpack_done", "unused", "acc_last", "epi_done", "upstream_done", "mma_last"]


def main():
    import bench
    from gridllm_b200 import native as N
    path = bench.build_model_once("llama3_8b_q4km", 0, lambda: None)
    batch = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    ctx = int(sys.argv[2]) if len(sys.argv) > 2 else 576
    e = N.Engine(path, max_ctx=1024, max_batch=max(2, batch), batch_weights=2)
    lib = N.load_library()
    fn = lib.gl_dbg_qgemm_trace
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
    ms0, _, _ = e.time_batch_step(batch, ctx, 2)      # builds the batch state (its un-captured warm pass uses trace slots too)
    fn(None, 0, 1)                                   # forget everything so far
    # a fresh bucket would reuse the captured graph: force a new capture by asking for another engine
    e.close()
    e = N.Engine(path, max_ctx=1024, max_batch=max(2, batch), batch_weights=2)
    fn(None, 0, 1)
    ms, nl, _ = e.time_batch_step(batch, ctx, 4)
    n = fn(None, 0, 0)
    buf = np.zeros((n, GRID, SLOTS), np.uint64)
    fn(buf.ctypes.data_as(ctypes.c_void_p), n, 0)
    print({"batch": batch, "ctx": ctx, "ms_per_step": ms, "qgemm_launch_slots": n})
    # the last 129 traced launches with data are the captured step (warm pass first, capture after)
    live = [i for i in range(n) if buf[i, :, 0].max() > 0]
    step = live[-129:]
    t = buf[step].astype(np.int64)
    order = np.argsort([tt[:, 0][tt[:, 0] > 0].min() for tt in t])
    t = t[order]
    rows = []
    for k, tt in enumerate(t):
        m = tt[:, 0] > 0
        base = tt[m, 0].min()
        rel = (tt[m] - base) / 1e3
        end = rel[:, 7].max()
        nxt = (t[k + 1][:, 0][t[k + 1][:, 0] > 0].min() - base) / 1e3 if k + 1 < len(t) else float("nan")
        rows.append(dict(ctas=int(m.sum()), entry_max=rel[:, 0].max(), prologue=np.median(rel[:, 1]), tma0=np.median(rel[:, 2]),
                         upstream=np.median(rel[:, 8]), qtile0=np.median(rel[:, 3]), unpack_med=np.median(rel[:, 4]),
                         unpack_max=rel[:, 4].max(), mma_last=np.median(rel[:, 9]), acc_med=np.median(rel[:, 6]),
                         acc_max=rel[:, 6].max(), epi_med=np.median(rel[:, 7]), end=end, next_entry=nxt))
    keys = list(rows[0].keys())
    print("launch  " + " ".join("%11s" % k for k in keys))
    for k in list(range(0, 8)) + [len(rows) - 1]:
        print("%6d  " % k + " ".join("%11.2f" % rows[k][kk] for kk in keys))
    print("mean over layers 1..31 by position in the layer (0 QKV, 1 attn_output, 2 gate/up, 3 ffn_down):")
    for pos in range(4):
        sel = [rows[4 * l + pos] for l in range(1, 32)]
        print("%6s  " % ("p%d" % pos) + " ".join("%11.2f" % np.mean([r[kk] for r in sel]) for kk in keys))
    e.close()


if __name__ == "__main__":
    main()
