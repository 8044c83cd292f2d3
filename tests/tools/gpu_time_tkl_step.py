"""Where one TKL bench step spends its time on the GPU box: every component between CUDA events (test tooling)."""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bench  # noqa: E402
from matchmaker_b200 import interaction  # noqa: E402

dev = torch.device("cuda", 0)
wl = bench.TklWorkload(0, dev)
wl.to_device()
c = wl.c


def timed(name, fn, n=30):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    print(f"{name:34s} gpu {e0.elapsed_time(e1) / n * 1e3:8.1f} us   host-issue {(time.perf_counter() - t0) / n * 1e6:8.1f} us", flush=True)


timed("slot map", lambda: interaction._tkl_slot_map(c["pk"]))
ws_holder = {}


def win(impl):
    ws_holder["ws"] = interaction.tkl_window_scores(c["q"], c["qm"], c["ch"], c["cm"], c["pk"], wl.pieces, c["mu"], c["sg"], c["dw"],
                                                    "embedding", c["sat"], c["red"], impl=impl)


timed("window scores (auto)", lambda: win("auto"))
timed("window scores (tensor cores)", lambda: win("tcgen05"))
timed("window scores (simt)", lambda: win("simt"), n=5)
timed("top hills", lambda: interaction.tkl_top_hills(ws_holder["ws"], c["cs"]))
timed("full step", wl.kernel_step)
g = bench.graphed_step(wl.kernel_step, dev)
if g is not None:
    timed("full step (CUDA graph replay)", g)
