"""The TK training step's interaction (ecai20_tk.py:105-124: cosine, RBF kernels, masked sums, log, linear) over
BERT-width embeddings on one GPU: autograd.kernel_pool (the saving tensor-core forward, then the wide tensor-core backward
of csrc/kernel_pool_wide.cu) against the reference's torch expression (oracle.kernel_pool_tk) with torch autograd on the
same GPU, and the kernels alone.

64 pairs, Lq 30 with query lengths 5-30, Ld 200 with lengths 50-200, TK's 11 kernels with alpha, fp32, at D 768 (BERT-base)
and 1024 (BERT-large).  Per path: forward + backward time per step (CUDA-event medians over alternated rounds after
warm-up; each window holds --steps steps), and the peak memory of one step above the inputs.  For the kernels alone: the
training forward (interaction.kernel_pool with save_for_backward) and the backward (interaction.kernel_pool_bwd with the
saved state), each timed on its own, and the backward's bytes over its time against the H100 SXM's 3.35 TB/s.  The
bytes are those the backward has to move: q, d, the saved state and S read, grad_q and grad_d written.  The workspace
holding G is not counted.  Also the worst gradient difference between the two paths, max |a - b| / max |b| per input.

    python scripts/bench_kernel_pool_wide.py --out-dir DIR
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_colbert_e2e import power_limit_w, summary  # noqa: E402
from matchmaker_b200 import autograd, interaction  # noqa: E402
from oracle import interaction_oracle as O  # noqa: E402

HBM_PEAK_BPS = 3.35e12   # H100 SXM data sheet


def sm_clock_mhz():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def make_batch(args, D, dev):
    g = torch.Generator(device=dev).manual_seed(D)
    B, Lq, Ld = args.batch, args.lq, args.ld
    q = torch.randn(B, Lq, D, generator=g, device=dev).requires_grad_(True)
    d = torch.randn(B, Ld, D, generator=g, device=dev).requires_grad_(True)
    qm = (torch.arange(Lq, device=dev).unsqueeze(0) < torch.randint(5, Lq + 1, (B, 1), generator=g, device=dev)).float()
    dm = (torch.arange(Ld, device=dev).unsqueeze(0) < torch.randint(50, Ld + 1, (B, 1), generator=g, device=dev)).float()
    mu, sigma = (torch.tensor(v, device=dev) for v in ([1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9], [0.1] * 11))
    weight = ((torch.rand(11, generator=g, device=dev) - 0.5) * 0.028).requires_grad_(True)
    alpha = (torch.rand(11, generator=g, device=dev) + 0.5).requires_grad_(True)
    gout = torch.randn(B, generator=g, device=dev)
    return dict(q=q, d=d, qm=qm, dm=dm, mu=mu, sigma=sigma, weight=weight, alpha=alpha, gout=gout)


def kernel_step(x):
    score, _ = autograd.kernel_pool(x["q"], x["d"], x["qm"], x["dm"], x["mu"], x["sigma"], x["weight"], x["alpha"], 1.0)
    return score


def torch_step(x):
    score, _ = O.kernel_pool_tk(x["q"], x["d"], x["qm"], x["dm"], x["mu"], x["sigma"], x["alpha"], x["weight"])
    return score


PATHS = {"kernel": kernel_step, "torch": torch_step}
LEAVES = ("q", "d", "weight", "alpha")


def steps(path, x, k):
    """k forward + backward steps back to back; seconds per step."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(k):
        for n in LEAVES:
            x[n].grad = None
        (PATHS[path](x) * x["gout"]).sum().backward()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e-3 / k


def kernels_alone(x, k):
    """The training forward and the backward entry points, each timed over k calls; seconds per call."""
    args = [x[n].detach() for n in ("q", "d", "qm", "dm", "mu", "sigma", "weight")]
    alpha = x["alpha"].detach()

    def fwd():
        return interaction.kernel_pool(*args, alpha=alpha, log_scale=1.0, want_per_kernel=True, save_for_backward=True)

    out = fwd()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    for _ in range(k):
        fwd()
    ev[1].record()
    for _ in range(k):
        interaction.kernel_pool_bwd(*args, alpha, out["per_kernel_query"], x["gout"], 1.0, saved=out["saved"])
    ev[2].record()
    ev[2].synchronize()
    return ev[0].elapsed_time(ev[1]) * 1e-3 / k, ev[1].elapsed_time(ev[2]) * 1e-3 / k


def backward_bytes(B, Lq, Ld, D, K):
    inputs = B * Lq * D + B * Ld * D + B * (33 * Ld + 32) + B * Lq * K
    outputs = B * Lq * D + B * Ld * D
    return 4 * (inputs + outputs)


def run_dim(args, D, dev):
    x = make_batch(args, D, dev)
    res = {"dim": D}
    got = {}
    for path in PATHS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        steps(path, x, 1)
        res[f"{path}_peak_mem_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        got[path] = [x[n].grad.clone() for n in LEAVES]
    res["worst_grad_diff_over_scale"] = {n: ((a - b).abs().max() / b.abs().max()).item()
                                         for n, a, b in zip(LEAVES, got["kernel"], got["torch"])}
    for path in PATHS:
        steps(path, x, args.warmup)
    kernels_alone(x, args.warmup)
    times = {p: [] for p in PATHS}
    fwd, bwd = [], []
    for r in range(args.rounds):
        for path in (list(PATHS) if r % 2 == 0 else list(PATHS)[::-1]):
            times[path].append(steps(path, x, args.steps))
        f, b = kernels_alone(x, args.steps)
        fwd.append(f)
        bwd.append(b)
    for path in PATHS:
        res[f"{path}_step"] = summary(times[path])
    res["kernel_forward_alone"] = summary(fwd)
    res["kernel_backward_alone"] = summary(bwd)
    res["step_speedup"] = res["torch_step"]["median_s"] / res["kernel_step"]["median_s"]
    nbytes = backward_bytes(args.batch, args.lq, args.ld, D, 11)
    res["backward_bytes"] = nbytes
    res["backward_bytes_per_s"] = nbytes / res["kernel_backward_alone"]["median_s"]
    res["backward_share_of_hbm_peak"] = res["backward_bytes_per_s"] / HBM_PEAK_BPS
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--lq", type=int, default=30)
    ap.add_argument("--ld", type=int, default=200)
    ap.add_argument("--dims", type=int, nargs="+", default=[768, 1024])
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10, help="steps per timed window")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kernel_pool_wide.py measures on a GPU; none is available")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    props = torch.cuda.get_device_properties(dev)
    out = {"gpu": props.name, "power_limit_w": power_limit_w(), "max_sm_clock_mhz": sm_clock_mhz(), "batch": args.batch,
           "lq": args.lq, "ld": args.ld, "kernels": 11, "dtype": "float32", "steps_per_window": args.steps,
           "results": [run_dim(args, D, dev) for D in args.dims]}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, "bench_kernel_pool_wide.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
