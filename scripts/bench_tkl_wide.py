"""TKL training at BERT widths on one GPU: the interaction step (autograd forward + backward) and the backward alone.

    python scripts/bench_tkl_wide.py [--reps 7] [--iters 10] [--out results.json]

Shape: K 11 kernels, Lq 30, max_doc_length 2000, documents of 200-2000 tokens (mean ~1 100), 16 and 128 documents, both
saturations, at D 768 and 1024.  For each it reports:
  * the kernel path: autograd.tkl_interaction forward + backward, and interaction.tkl_bwd_wide alone on the same windows;
  * the oracle expression (oracle.interaction_oracle.tkl_interaction) in fp32 torch on the same GPU, forward + backward;
  * the backward's bytes over its time against 3.35 TB/s (the H100 SXM data-sheet HBM3 rate), and peak memory.
At D 300 it also times tkl_bwd_wide against the one-CTA-per-document tkl_bwd.  Times are medians over alternated
windows of ``--iters`` calls each, measured with CUDA events.  The card's name and power limit are printed with them.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from matchmaker_b200 import autograd, interaction  # noqa: E402
from matchmaker_b200.rankers.tkl import chunk_documents  # noqa: E402
from oracle import interaction_oracle as O  # noqa: E402

HBM_BPS = 3.35e12
K, LQ, MAX_LEN = 11, 30, 2000
MU = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]
SIGMA = [0.001] + [0.1] * 10


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, limit = torch.cuda.get_device_name(0), "unknown"
    return name, limit


def make(B, D, sat, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(200, MAX_LEN + 1, (B,), generator=g)
    q = torch.randn(B, LQ, D, generator=g) * 0.4
    d = torch.randn(B, MAX_LEN, D, generator=g) * 0.4
    dm = (torch.arange(MAX_LEN).unsqueeze(0) < lens.unsqueeze(1)).float()
    qm = torch.ones(B, LQ)
    dev = "cuda"
    q, d, qm, dm = q.to(dev), (d * dm.unsqueeze(-1)).to(dev), qm.to(dev), dm.to(dev)
    cd2, cm2, packed, pieces = chunk_documents(d, dm)
    chunks = cd2[packed][:, 5:-5].contiguous()
    cmask = cm2[packed][:, 5:-5].contiguous()
    p = {"mu": torch.tensor(MU, device=dev), "sigma": torch.tensor(SIGMA, device=dev),
         "dense_weight": torch.randn(K, generator=g).to(dev) * 0.1, "chunk_scoring": torch.rand(15, generator=g).to(dev),
         "sat_emb_reduce1_weight": (torch.randn(D, generator=g) * 0.03).to(dev),
         "sat_normer_weight": torch.ones(2, device=dev), "sat_normer_bias": torch.zeros(2, device=dev),
         "saturation_linear_weight": torch.full((2,), 0.01, device=dev), "saturation_linear_bias": torch.tensor([3.], device=dev),
         "saturation_linear2_weight": torch.full((2,), 0.01, device=dev), "saturation_linear2_bias": torch.tensor([2.], device=dev),
         "saturation_linear3_weight": torch.full((2,), 0.01, device=dev), "saturation_linear3_bias": torch.tensor([1.], device=dev),
         "kernel_mult0": torch.ones(K, device=dev)}
    if sat == "embedding":
        keys = ("sat_normer_weight", "sat_normer_bias", "saturation_linear_weight", "saturation_linear_bias",
                "saturation_linear2_weight", "saturation_linear2_bias", "saturation_linear3_weight",
                "saturation_linear3_bias")
        sp, red = torch.cat([p[k].reshape(-1) for k in keys]), p["sat_emb_reduce1_weight"]
    else:
        sp, red = p["kernel_mult0"], None
    return dict(q=q, qm=qm, chunks=chunks, cmask=cmask, packed=packed, pieces=pieces, p=p, sp=sp, red=red,
                gout=torch.randn(B, generator=g).to(dev), lens=lens)


def kernel_step(c, sat):
    q = c["q"].requires_grad_(True)
    ch = c["chunks"].requires_grad_(True)
    score, *_ = autograd.tkl_interaction(q, c["qm"], ch, c["cmask"], c["packed"], c["pieces"], c["p"]["mu"],
                                         c["p"]["sigma"], c["p"]["dense_weight"], sat, c["sp"], c["red"],
                                         c["p"]["chunk_scoring"])
    torch.autograd.grad((score * c["gout"]).sum(), (q, ch))


def oracle_step(c, sat):
    q = c["q"].requires_grad_(True)
    ch = c["chunks"].requires_grad_(True)
    with torch.device("cuda"):   # the oracle's own temporaries follow the default device
        score, _ = O.tkl_interaction(q, c["qm"], ch, c["cmask"], c["packed"], c["pieces"], c["p"], sat)
    torch.autograd.grad((score * c["gout"]).sum(), (q, ch))


def bwd_args(c, sat):
    ws = interaction.tkl_window_scores(c["q"], c["qm"], c["chunks"], c["cmask"], c["packed"], c["pieces"], c["p"]["mu"],
                                       c["p"]["sigma"], c["p"]["dense_weight"], sat, c["sp"], c["red"])
    _, orig, top_idx, _ = interaction.tkl_top_hills(ws, c["p"]["chunk_scoring"])
    return (c["q"].detach(), c["qm"], c["chunks"].detach(), c["cmask"], c["packed"], c["pieces"], c["p"]["mu"],
            c["p"]["sigma"], c["p"]["dense_weight"], sat, c["sp"], c["red"], c["p"]["chunk_scoring"], top_idx, orig,
            c["gout"])


def bwd_bytes(c, D):
    """HBM bytes the wide backward must move, from shapes: the zero fill of grad_chunks, q and the <= 114 union rows read
    twice (dot and grad kernels), grad_q and the union's gradient rows written, the workspace records written and read."""
    B, nc = c["q"].shape[0], c["chunks"].shape[0]
    rows = B * 114
    rec = 40 * 128 + 208
    nb = (D + 63) // 64
    return 4 * (nc * 40 * D + 2 * (B * LQ * D + rows * D) + B * LQ * D + rows * D + 2 * B * (nb + 1) * rec)


def timed(fns, reps, iters):
    """Median ms per call of each fn over ``reps`` alternated windows of ``iters`` calls."""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    res = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                f()
            b.record()
            b.synchronize()
            res[k].append(a.elapsed_time(b) / iters)
    return {k: statistics.median(v) for k, v in res.items()}


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2**20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tkl_wide.py needs a GPU")
    name, limit = card()
    rows = []
    for D in (768, 1024):
        for B in (16, 128):
            for sat in ("embedding", "log"):
                c = make(B, D, sat, seed=D + B)
                ba = bwd_args(c, sat)
                t = timed({"step": lambda: kernel_step(c, sat), "bwd": lambda: interaction.tkl_bwd_wide(*ba),
                           "oracle_step": lambda: oracle_step(c, sat)}, args.reps, args.iters)
                nbytes = bwd_bytes(c, D)
                row = {"D": D, "B": B, "sat": sat, "mean_doc_len": float(c["lens"].float().mean()),
                       "step_ms": t["step"], "bwd_ms": t["bwd"], "oracle_step_ms": t["oracle_step"],
                       "oracle_over_kernel": t["oracle_step"] / t["step"],
                       "bwd_bytes": nbytes, "bwd_TBps": nbytes / t["bwd"] / 1e9, "bwd_of_hbm": nbytes / (t["bwd"] * 1e-3) / HBM_BPS,
                       "peak_MiB_step": peak(lambda: kernel_step(c, sat)),
                       "peak_MiB_oracle": peak(lambda: oracle_step(c, sat))}
                rows.append(row)
                print(json.dumps(row), flush=True)
    for B in (16, 128):
        for sat in ("embedding", "log"):
            c = make(B, 300, sat, seed=300 + B)
            ba = bwd_args(c, sat)
            t = timed({"wide": lambda: interaction.tkl_bwd_wide(*ba), "one_cta": lambda: interaction.tkl_bwd(*ba)},
                      args.reps, args.iters)
            row = {"D": 300, "B": B, "sat": sat, "wide_bwd_ms": t["wide"], "one_cta_bwd_ms": t["one_cta"]}
            rows.append(row)
            print(json.dumps(row), flush=True)
    summary = {"card": name, "power_limit": limit, "rows": rows}
    print(json.dumps({"card": name, "power_limit": limit}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
