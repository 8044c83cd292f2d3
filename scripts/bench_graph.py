"""Graph index against exact search and IVF on one shard of the reference's dense-retrieval shape.

    python scripts/bench_graph.py [--rows 1100000] [--dim 768] [--queries 6400] [--M 32 64] [--ef-search 64 128 256 512]

Two seeded synthetic sets, fp16 storage: bench_ivf.py's clustered set (well-separated clusters) and an overlapping set
whose noise is four times as long as the unit cluster centres.  For each set: the k-NN graph is built once (K = max(2M,
efConstruction) is 128 for both M at efConstruction 128) and pruned and merged for every M.  Reports the build time
split into k-NN, prune and reverse/merge; per efSearch the device time of each search stage (entry scan, beam search)
from torch.profiler and the CUDA-event end-to-end time; recall@top_n against FlatIPIndexer; the gathered-row bytes/s and
its share of HBM; and IVF at several nprobe on the same data, to compare at matched recall.  Rows gathered per query
are counted by replaying the beam search of the first --visit-queries queries on the host with an exact visited set; the
bytes/s figure scales their mean to all queries.  Prints the card and its power limit.  One JSON line on stdout.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_ivf import HBM_BYTES_PER_S, clustered, kernel_ms, power_limit_w, timed  # noqa: E402
from matchmaker_b200 import _lib, interaction  # noqa: E402
from matchmaker_b200.retrieval import FlatIPIndexer, GraphIndexer, IVFIndexer  # noqa: E402
from matchmaker_b200.retrieval import graph_index  # noqa: E402

STAGES = {"flat_ip_tc_kernel": "entry_scan", "topk_merge_kernel": "entry_scan", "graph_search_kernel": "beam_search"}


def overlapping(n, dim, n_clusters, nq, seed, dev, spread=4.0):
    """Clusters whose noise is longer than the distance between centres, so that the k-NN graph joins them (with
    bench_ivf's spread of 0.5, or even 1.0, in 768 dimensions every cluster stays a component of its own)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    centers = torch.nn.functional.normalize(torch.randn(n_clusters, dim, generator=g, device=dev), dim=1)
    x = torch.empty(n, dim, dtype=torch.float16, device=dev)
    for lo in range(0, n, 1 << 18):
        hi = min(n, lo + (1 << 18))
        lab = torch.randint(0, n_clusters, (hi - lo,), generator=g, device=dev)
        x[lo:hi] = (centers[lab] + spread * torch.randn(hi - lo, dim, generator=g, device=dev) / dim ** 0.5).half()
    ql = torch.randint(0, n_clusters, (nq,), generator=g, device=dev)
    q = (centers[ql] + spread * torch.randn(nq, dim, generator=g, device=dev) / dim ** 0.5).half()
    return x, q


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def rows_visited(idx, q, L, n_queries):
    """Distinct rows the beam search scores for the first n_queries queries: a host replay with an exact visited set
    (scores from the same fp16 rows in fp32; near-ties may order differently from the kernel, so this is a count)."""
    graph = idx.graph.cpu().numpy()
    ent = idx.entries(q[:n_queries], L).cpu().numpy()
    out = []
    for a in range(n_queries):
        qa = q[a].float()
        score = dict(zip(ent[a].tolist(), (idx.rows[torch.from_numpy(ent[a]).to(q.device)].float() @ qa).tolist()))
        lst = sorted(score, key=lambda p: (-score[p], p))[:L]
        parents = set()
        for _ in range(2 * L):
            cand = [p for p in lst if p not in parents]
            if not cand:
                break
            parents.add(cand[0])
            new = [int(v) for v in graph[cand[0]] if v >= 0 and int(v) not in score]
            if new:
                s = (idx.rows[torch.tensor(new, device=q.device)].float() @ qa).tolist()
                score.update(zip(new, s))
                lst = sorted(lst + new, key=lambda p: (-score[p], p))[:L]
        out.append(len(score))
    return out


def recall(got, exact, k):
    return float(np.mean([len(set(a) & set(b)) / k for a, b in zip(got.tolist(), exact.tolist())]))


def run_set(name, x, q, args, res):
    dev = x.device
    n, dim, k = x.shape[0], x.shape[1], args.top_n
    ids = np.arange(n, dtype=np.int64)
    xh = x.cpu().numpy()
    out = {"builds": {}, "search": {}, "ivf": {}}
    cfg = {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_hnsw_efConstruction": args.ef_construction,
           "faiss_hnsw_efSearch": args.ef_search[0], "faiss_ivf_list_count": args.nlist, "faiss_ivf_search_probe_count": 1}
    flat = FlatIPIndexer(cfg)
    flat.index([ids], [xh])
    out["flat_ms"] = timed(lambda: flat.search_device(q, k), args.reps, args.warmup)
    _, exact = flat.search_device(q, k)

    knn_cache = {}
    for M in args.M:
        idx = GraphIndexer(dict(cfg, faiss_hnsw_graph_neighbors=M))
        idx.rows, idx.ids = x, torch.from_numpy(ids).to(dev)
        if idx.K not in knn_cache:
            knn_cache[idx.K] = wall(lambda: graph_index.knn_graph(x, idx.K))
        knn, knn_s = knn_cache[idx.K]
        pruned, prune_s = wall(lambda: interaction.graph_prune(knn, idx.R))
        idx.graph, merge_s = wall(lambda: graph_index.reverse_merge(pruned))
        idx._set_entries(torch.from_numpy(graph_index.entry_positions(n)).to(dev))
        deg = (idx.graph >= 0).sum(1).float()
        out["builds"][str(M)] = {"R": idx.R, "K": idx.K, "knn_s": knn_s, "prune_s": prune_s, "merge_s": merge_s,
                                 "knn_flop": 2.0 * n * n * dim, "mean_degree": float(deg.mean()),
                                 "entries": int(idx.entry_pos.numel())}
        for efs in args.ef_search:
            idx.ef_search = efs
            L = graph_index.search_list_size(efs, k)
            total_ms = timed(lambda: idx.search_device(q, k), args.reps, args.warmup)
            stages = kernel_ms(lambda: idx.search_device(q, k), args.reps, STAGES)
            _, got = idx.search_device(q, k)
            counts = rows_visited(idx, q, L, args.visit_queries)
            visited = float(np.mean(counts))
            gathered = visited * q.shape[0] * (dim * 2 + idx.R * 4)   # row bytes plus its neighbour list
            out["search"][f"{M}/{efs}"] = {
                "L": L, "total_ms": total_ms, "entry_scan_ms": stages["entry_scan"], "beam_search_ms": stages["beam_search"],
                "recall_at_top_n": recall(got, exact, k), "speedup_vs_flat": out["flat_ms"] / total_ms,
                "rows_visited_per_query": visited, "rows_visited_min_max": [min(counts), max(counts)],
                "rows_visited_queries": len(counts),
                "gathered_bytes_per_s": gathered / (stages["beam_search"] * 1e-3),
                "gathered_hbm_share": gathered / (stages["beam_search"] * 1e-3) / HBM_BYTES_PER_S}
        del idx
    del knn_cache
    ivf = IVFIndexer(cfg)
    _, out["ivf_train_s"] = wall(lambda: ivf.prepare([xh]))
    ivf.index([ids], [xh])
    for nprobe in args.nprobe:
        ivf.nprobe = nprobe
        t = timed(lambda: ivf.search_device(q, k), args.reps, args.warmup)
        _, got = ivf.search_device(q, k)
        out["ivf"][str(nprobe)] = {"total_ms": t, "recall_at_top_n": recall(got, exact, k)}
    res["sets"][name] = out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_100_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--queries", type=int, default=6400)
    ap.add_argument("--top-n", type=int, default=100)
    ap.add_argument("--M", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--ef-construction", type=int, default=128)
    ap.add_argument("--ef-search", type=int, nargs="+", default=[64, 128, 256, 512])
    ap.add_argument("--clusters", type=int, default=5000)
    ap.add_argument("--nlist", type=int, default=20000)
    ap.add_argument("--nprobe", type=int, nargs="+", default=[5, 10, 20, 50, 100])
    ap.add_argument("--sets", nargs="+", default=["clustered", "overlapping"])
    ap.add_argument("--visit-queries", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "rows": args.rows, "dim": args.dim,
           "queries": args.queries, "top_n": args.top_n, "ef_construction": args.ef_construction, "sets": {}}
    for name in args.sets:
        gen = clustered if name == "clustered" else overlapping
        x, q = gen(args.rows, args.dim, args.clusters, args.queries, 0, dev)
        run_set(name, x, q, args, res)
        del x, q
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    _lib.load()
    main()
