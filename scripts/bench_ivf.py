"""IVF index against exact search on one shard of the reference's dense-retrieval shape.

    python scripts/bench_ivf.py [--rows 1100000] [--dim 768] [--queries 6400] [--nlist 20000] [--nprobe 50 100 500]

A seeded clustered synthetic set (fp16 storage), the shape of one 1.1 M-passage shard with 6 400 queries and the
reference's example IVF config (20 000 lists).  Reports training and add time, per-stage search times (coarse,
inversion + gather, scan, merge) as CUDA-event medians after warm-up, recall@top_n against FlatIPIndexer and the speedup
over it, the scan's bytes/s and its share of HBM bandwidth, where the training time goes, the card and its power limit.
The stage times of one ivf_search call are the device times of its kernels (torch.profiler).  One JSON line on stdout.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from matchmaker_b200 import _lib, interaction  # noqa: E402
from matchmaker_b200.retrieval import FlatIPIndexer, IVFIndexer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def clustered(n, dim, n_clusters, nq, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    centers = torch.nn.functional.normalize(torch.randn(n_clusters, dim, generator=g, device=dev), dim=1)
    x = torch.empty(n, dim, dtype=torch.float16, device=dev)
    for lo in range(0, n, 1 << 18):
        hi = min(n, lo + (1 << 18))
        lab = torch.randint(0, n_clusters, (hi - lo,), generator=g, device=dev)
        x[lo:hi] = (centers[lab] + 0.5 * torch.randn(hi - lo, dim, generator=g, device=dev) / dim ** 0.5).half()
    ql = torch.randint(0, n_clusters, (nq,), generator=g, device=dev)
    q = (centers[ql] + 0.5 * torch.randn(nq, dim, generator=g, device=dev) / dim ** 0.5).half()
    return x, q


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


# kernel name -> search stage of one ivf_search call
STAGES = {"ivf_count_kernel": "inversion_gather", "ivf_scan_kernel": "inversion_gather",
          "ivf_gather_kernel": "inversion_gather", "ivf_items_kernel": "inversion_gather", "fill_u32": "inversion_gather",
          "Memset": "inversion_gather", "flat_ip_tc_kernel": "scan", "topk_merge_kernel": "merge"}


def kernel_ms(fn, reps, stages):
    """Device time per call of the kernels fn() launches, summed per stage (torch.profiler, CUDA activity only)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {v: 0.0 for v in stages.values()}
    for e in prof.key_averages():
        for needle, stage in stages.items():
            if needle in e.key:
                out[stage] += getattr(e, "device_time_total", 0.0) / 1e3 / reps
                break
    return out


def train_breakdown(ivf, xh, reps, warmup):
    """Where one k-means iteration spends its time, at the trained centroids: loading the training points, the
    assignment (flat_ip_topk with k = 1), the stable sort into lists, the list means and the empty-list split."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    x, _ = ivf._training_points([xh])
    torch.cuda.synchronize()
    out = {"load_points_s": time.perf_counter() - t0, "points": int(x.shape[0])}
    c = ivf.centroids
    store, scale = ivf._centroid_store(c)
    out["assign_ms"] = timed(lambda: interaction.flat_ip_topk(x, store, 1, split_scale=scale), reps, warmup)
    a = interaction.flat_ip_topk(x, store, 1, split_scale=scale)[1][:, 0]
    out["layout_ms"] = timed(lambda: ivf._layout(a), reps, warmup)
    perm, off = ivf._layout(a)
    out["list_means_ms"] = timed(lambda: interaction.ivf_list_means(x, perm, off), reps, warmup)
    ivf._counts = off[1:] - off[:-1]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _, n_split = ivf._split_empty(c, np.random.RandomState(0))
    torch.cuda.synchronize()
    out["split_ms"], out["empty_lists"] = (time.perf_counter() - t0) * 1e3, n_split
    out["iterations"], out["splits_per_iteration"] = len(ivf.train_splits), ivf.train_splits
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_100_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--queries", type=int, default=6400)
    ap.add_argument("--nlist", type=int, default=20000)
    ap.add_argument("--nprobe", type=int, nargs="+", default=[50, 100, 500])
    ap.add_argument("--top-n", type=int, default=100)
    ap.add_argument("--clusters", type=int, default=5000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    x, q = clustered(args.rows, args.dim, args.clusters, args.queries, 0, dev)
    xh = x.cpu().numpy()
    ids = np.arange(args.rows, dtype=np.int64)
    cfg = {"token_dim": args.dim, "faiss_use_gpu": True, "token_dtype": "float16",
           "faiss_ivf_list_count": args.nlist, "faiss_ivf_search_probe_count": args.nprobe[0]}
    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "rows": args.rows, "dim": args.dim,
           "queries": args.queries, "nlist": args.nlist, "top_n": args.top_n, "runs": {}}

    flat = FlatIPIndexer(cfg)
    flat.index([ids], [xh])
    res["flat_ms"] = timed(lambda: flat.search_device(q, args.top_n), args.reps, args.warmup)
    _, exact = flat.search_device(q, args.top_n)

    ivf = IVFIndexer(cfg)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ivf.prepare([xh])
    torch.cuda.synchronize()
    res["train_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    ivf.index([ids], [xh])
    torch.cuda.synchronize()
    res["add_s"] = time.perf_counter() - t0
    res["train_breakdown"] = train_breakdown(ivf, xh, args.reps, args.warmup)
    sizes = (ivf.list_offsets[1:] - ivf.list_offsets[:-1]).float()
    res["list_len_mean"], res["list_len_max"] = float(sizes.mean()), int(sizes.max())

    row_bytes = ivf.rows.shape[1] * 2
    for nprobe in args.nprobe:
        ivf.nprobe = nprobe
        probes = ivf.coarse(q)
        coarse_ms = timed(lambda: ivf.coarse(q), args.reps, args.warmup)
        call = lambda: interaction.ivf_search(q, ivf.rows, ivf.ids, ivf.list_offsets, probes, args.top_n,  # noqa: E731
                                              ivf.max_list_len)
        call_ms = timed(call, args.reps, args.warmup)
        total_ms = timed(lambda: ivf.search_device(q, args.top_n), args.reps, args.warmup)
        stages = kernel_ms(call, args.reps, STAGES)
        _, got = ivf.search_device(q, args.top_n)
        recall = float(np.mean([len(set(a) & set(b)) / args.top_n for a, b in zip(got.tolist(), exact.tolist())]))
        lens = (ivf.list_offsets[probes + 1] - ivf.list_offsets[probes])
        # every list is read once per chunk of <= 128 queries probing it
        probed = torch.bincount(probes.reshape(-1), minlength=ivf.nlist)
        chunks = (probed + 127) // 128
        bytes_read = float(((ivf.list_offsets[1:] - ivf.list_offsets[:-1]) * chunks).sum()) * row_bytes
        scan_kernel_ms = stages["scan"]
        res["runs"][str(nprobe)] = {
            "coarse_ms": coarse_ms, "inversion_gather_ms": stages["inversion_gather"], "scan_ms": scan_kernel_ms,
            "merge_ms": stages["merge"], "ivf_search_call_ms": call_ms, "total_ms": total_ms, "recall_at_top_n": recall,
            "speedup_vs_flat": res["flat_ms"] / total_ms, "rows_scanned_per_query": float(lens.sum(1).float().mean()),
            "scan_bytes_per_s": bytes_read / (scan_kernel_ms * 1e-3),
            "scan_hbm_share": bytes_read / (scan_kernel_ms * 1e-3) / HBM_BYTES_PER_S}
    print(json.dumps(res))


if __name__ == "__main__":
    _lib.load()
    main()
