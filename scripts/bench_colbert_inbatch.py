"""Training-time in-batch scoring of ColBERT (in-batch negatives, colbert.py:154-162) on one GPU: the differentiable
all-pairs max-sim (autograd.maxsim_allpairs: the argmax forward, then mmb200_maxsim_allpairs_bwd) against the reference
expression in torch (oracle.maxsim_allpairs: mm, mask, max, sum, with torch autograd on the GPU).

The batch is TAS-B's (batch_size_train 32): 32 queries x 32 positive and 32 negative passages, i.e. two all-pairs calls
of 1 024 pairs, fp16, Lq 32 with query lengths 5-32, Ld 200 with MSMARCO-shaped passage lengths (about 75 +- 30 tokens),
at dim 768 (colbert.yaml) and dim 128. Both paths use the reference mask indexing. Per path: forward time, backward time
(CUDA-event medians over alternated rounds after warm-up; each window holds --steps steps, forwards back to back and
then their backwards, and reports the time per step), the backward kernels alone through
interaction.maxsim_allpairs_bwd, peak memory of one forward + backward above the inputs, and the worst gradient
difference between the paths (max |a - b| / max |b| per input), and of each path against the reference expression in
fp32 on the same fp16 inputs.

    python scripts/bench_colbert_inbatch.py --out-dir DIR
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_colbert_e2e import power_limit_w, summary  # noqa: E402
from matchmaker_b200 import autograd, interaction  # noqa: E402
from oracle import interaction_oracle as O  # noqa: E402


def make_batch(args, dim, dev, g):
    B, Lq, Ld = args.batch, args.lq, args.ld

    def vecs(n, L):
        return (torch.randn(n, L, dim, generator=g, device=dev) * (dim ** -0.5)).half().requires_grad_(True)

    q = vecs(B, Lq)
    qm = (torch.arange(Lq, device=dev).unsqueeze(0) < torch.randint(5, Lq + 1, (B, 1), generator=g, device=dev)).long()
    docs = []
    for _ in range(2):   # positives, negatives
        lens = torch.clamp(torch.round(torch.randn(B, 1, generator=g, device=dev) * 30 + 75), 10, Ld).long()
        docs.append((vecs(B, Ld), (torch.arange(Ld, device=dev).unsqueeze(0) < lens).long()))
    grads = [torch.randn(B, B, generator=g, device=dev) for _ in range(2)]
    return q, qm, docs, grads


def kernel_scores(q, qm, docs):
    return [autograd.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=True) for d, dm in docs]


def torch_scores(q, qm, docs):
    return [O.maxsim_allpairs(q, qm, d, dm) for d, dm in docs]


PATHS = {"kernel": kernel_scores, "torch": torch_scores}


def steps(path, q, qm, docs, grads, k):
    """k forwards back to back, then the k backwards; returns (forward s, backward s) per step.  A window of k steps
    keeps the device queue full, so a window does not close on host-side gaps between sub-millisecond launches."""
    for t in [q] + [d for d, _ in docs]:
        t.grad = None
    e = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    e[0].record()
    scores = [PATHS[path](q, qm, docs) for _ in range(k)]
    e[1].record()
    losses = [sum((s.float() * g).sum() for s, g in zip(sc, grads)) for sc in scores]
    e[2].record()
    for loss in losses:
        loss.backward()
    e[3].record()
    e[3].synchronize()
    return e[0].elapsed_time(e[1]) * 1e-3 / k, e[2].elapsed_time(e[3]) * 1e-3 / k


def backward_entry(q, qm, docs, grads, k):
    """The backward kernels alone (interaction.maxsim_allpairs_bwd, both calls of a step), k steps per window."""
    saved = []
    with torch.no_grad():
        for (d, dm), g in zip(docs, grads):
            _, am = interaction.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=True, return_argmax=True)
            saved.append((d.detach(), g, am))
    qd = q.detach()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(k):
        for d, g, am in saved:
            interaction.maxsim_allpairs_bwd(qd, d, g, am)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e-3 / k


def run_dim(args, dim, dev):
    g = torch.Generator(device=dev).manual_seed(dim)
    q, qm, docs, grads = make_batch(args, dim, dev, g)
    inputs = [q] + [d for d, _ in docs]
    res = {"dim": dim}
    got = {}
    for path in PATHS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        steps(path, q, qm, docs, grads, 1)
        res[f"{path}_peak_mem_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        got[path] = [t.grad.float().clone() for t in inputs]
    # the same fp16 inputs scored by the reference expression in fp32: where the two paths differ, this tells which
    # one moved (fp16 similarities in torch round near-tied maxima onto either row)
    q32 = q.detach().float().requires_grad_(True)
    docs32 = [(d.detach().float().requires_grad_(True), dm) for d, dm in docs]
    sum((s * g).sum() for s, g in zip(torch_scores(q32, qm, docs32), grads)).backward()
    got["fp32"] = [q32.grad] + [d.grad for d, _ in docs32]

    def worst(a, b):
        return {k: ((x - y).abs().max() / y.abs().max()).item() for k, x, y in zip(("q", "d_pos", "d_neg"), a, b)}

    res["worst_grad_diff_over_scale"] = worst(got["kernel"], got["torch"])
    res["kernel_vs_fp32_worst_grad_diff_over_scale"] = worst(got["kernel"], got["fp32"])
    res["torch_vs_fp32_worst_grad_diff_over_scale"] = worst(got["torch"], got["fp32"])
    for path in PATHS:
        steps(path, q, qm, docs, grads, args.warmup)
    backward_entry(q, qm, docs, grads, args.warmup)
    times = {p: ([], []) for p in PATHS}
    entry = []
    for r in range(args.rounds):
        order = list(PATHS) if r % 2 == 0 else list(PATHS)[::-1]
        for path in order:
            f, b = steps(path, q, qm, docs, grads, args.steps)
            times[path][0].append(f)
            times[path][1].append(b)
        entry.append(backward_entry(q, qm, docs, grads, args.steps))
    for path in PATHS:
        res[f"{path}_forward"] = summary(times[path][0])
        res[f"{path}_backward"] = summary(times[path][1])
    res["kernel_backward_entry_only"] = summary(entry)
    res["forward_speedup"] = res["torch_forward"]["median_s"] / res["kernel_forward"]["median_s"]
    res["backward_speedup"] = res["torch_backward"]["median_s"] / res["kernel_backward"]["median_s"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--lq", type=int, default=32)
    ap.add_argument("--ld", type=int, default=200)
    ap.add_argument("--dims", type=int, nargs="+", default=[768, 128])
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10, help="steps per timed window")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_colbert_inbatch.py measures on a GPU; none is available")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    props = torch.cuda.get_device_properties(dev)
    out = {"gpu": props.name, "power_limit_w": power_limit_w(), "batch": args.batch, "lq": args.lq, "ld": args.ld,
           "dtype": "float16", "mask_indexing": "reference", "steps_per_window": args.steps, "results": [run_dim(args, dim, dev) for dim in args.dims]}
    text = json.dumps(out, indent=1)
    print(text)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, "bench_colbert_inbatch.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
