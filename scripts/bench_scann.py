"""AH (faiss_index_type "scann") index against exact search and the IVF index on one shard of the reference's
dense-retrieval shape.

    python scripts/bench_scann.py [--rows 1100000] [--dim 768] [--queries 6400] [--batches 1 64 6400]

bench_ivf.py's seeded clustered set (fp16 storage, 1.1 M x 768 rows, 6 400 queries, top_n 100).  The AH index uses
its reference settings: int(sqrt(n)) leaves, min(100, nlist) probes, a shortlist of top_n rows re-scored exactly.  The
IVF index is built on the same leaves (the AH index's centroids) and probes as many; AH and IVF searches alternate in
the same run.  Reports the build time split into k-means, AH training and encoding, the index bytes, per-stage device
times of one search (torch.profiler), CUDA-event end-to-end medians per query batch size, recall@top_n against
FlatIPIndexer, the card and its power limit.  One JSON line on stdout.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from matchmaker_b200 import _lib  # noqa: E402
from matchmaker_b200.retrieval import FlatIPIndexer, IVFIndexer, ScaNNIndexer  # noqa: E402
from bench_ivf import clustered, kernel_ms, power_limit_w  # noqa: E402

# kernel name -> search stage (flat_ip_tc_kernel is the coarse stage of the AH search and the list scan of the IVF one)
AH_STAGES = {"flat_ip_tc_kernel": "coarse", "ivf_count_kernel": "inversion", "ivf_scan_kernel": "inversion",
             "ah_pairs_kernel": "inversion", "ivf_items_kernel": "inversion", "Memset": "inversion",
             "ah_scan_kernel": "code_scan", "topk_merge_kernel": "merge", "ah_reorder_kernel": "reorder",
             "elementwise": "torch_elementwise", "vectorized": "torch_elementwise"}
IVF_STAGES = {"flat_ip_tc_kernel": "coarse_and_scan", "ivf_count_kernel": "inversion_gather",
              "ivf_scan_kernel": "inversion_gather", "ivf_gather_kernel": "inversion_gather",
              "ivf_items_kernel": "inversion_gather", "fill_u32": "inversion_gather", "Memset": "inversion_gather",
              "topk_merge_kernel": "merge"}


def batched(fn, q, b):
    """fn over q in batches of b queries (the shape of a search loop with query_batch_size b)."""
    return lambda: [fn(q[i:i + b]) for i in range(0, q.shape[0], b)]


def median_ms(fn, reps, warmup):
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


def recall(got, exact, k):
    return float(np.mean([len(set(a) & set(b)) / k for a, b in zip(got.tolist(), exact.tolist())]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_100_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--queries", type=int, default=6400)
    ap.add_argument("--top-n", type=int, default=100)
    ap.add_argument("--clusters", type=int, default=5000)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 64, 6400])
    ap.add_argument("--batch1-queries", type=int, default=256, help="queries timed one by one at batch size 1")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    x, q = clustered(args.rows, args.dim, args.clusters, args.queries, 0, dev)
    xh = x.cpu().numpy()
    ids = np.arange(args.rows, dtype=np.int64)
    k = args.top_n
    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "rows": args.rows, "dim": args.dim,
           "queries": args.queries, "top_n": k}

    flat = FlatIPIndexer({"token_dim": args.dim, "faiss_use_gpu": True, "token_dtype": "float16"})
    flat.index([ids], [xh])
    _, exact = flat.search_device(q, k)

    ah = ScaNNIndexer({"token_dim": args.dim, "faiss_use_gpu": False, "token_dtype": "float16",
                       "query_sets": {"bench": {"top_n": k}}})
    t0 = time.perf_counter()
    ah.index([ids], [xh])
    torch.cuda.synchronize()
    res["ah_build_s"] = {"total": time.perf_counter() - t0, **ah.build_seconds}
    res["ah_train_loss"] = ah.train_loss
    res["nlist"], res["nprobe"] = ah.nlist, ah.nprobe
    res["ah_index_bytes"] = {"codes": ah.codes.numel(), "rows": ah.rows.numel() * 2, "ids": ah.ids.numel() * 8,
                             "centroids": ah.ivf.centroids.numel() * 4, "codebook": ah.codebook.numel() * 4}
    sizes = (ah.list_offsets[1:] - ah.list_offsets[:-1]).float()
    res["leaf_len_mean"], res["leaf_len_max"] = float(sizes.mean()), int(sizes.max())

    ivf = IVFIndexer({"token_dim": args.dim, "faiss_use_gpu": True, "token_dtype": "float16",
                      "faiss_ivf_list_count": ah.nlist, "faiss_ivf_search_probe_count": ah.nprobe})
    ivf.set_centroids(ah.ivf.centroids)
    ivf.index([ids], [xh])
    res["ivf_index_bytes"] = ivf.rows.numel() * 2 + ivf.ids.numel() * 8

    res["recall_at_top_n"] = {"ah": recall(ah.search_device(q, k)[1], exact, k),
                              "ivf": recall(ivf.search_device(q, k)[1], exact, k)}
    res["stages_ms_6400"] = {"ah": kernel_ms(lambda: ah.search_device(q, k), args.reps, AH_STAGES),
                             "ivf": kernel_ms(lambda: ivf.search_device(q, k), args.reps, IVF_STAGES)}
    res["end_to_end_ms"] = {}
    for b in args.batches:
        qq = q[:args.batch1_queries] if b == 1 else q
        row = {"queries": int(qq.shape[0])}
        for _ in range(2):   # AH and IVF alternate, twice
            for name, idx in (("ah", ah), ("ivf", ivf)):
                row.setdefault(name + "_ms", []).append(
                    median_ms(batched(lambda z, idx=idx: idx.search_device(z, k), qq, b), args.reps, args.warmup))
        row["ah_ms_per_query"] = float(np.median(row["ah_ms"])) / qq.shape[0]
        row["ivf_ms_per_query"] = float(np.median(row["ivf_ms"])) / qq.shape[0]
        res["end_to_end_ms"][str(b)] = row
    res["flat_ms_6400"] = median_ms(lambda: flat.search_device(q, k), args.reps, args.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    _lib.load()
    main()
