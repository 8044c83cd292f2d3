"""ColBERT IVF retrieval over the residual-compressed token store (retrieval.ColBERTResidualIndexer, b = 1 and 2)
against the uncompressed ColBERTIVFIndexer on one GPU, over bench_colbert_ivf.py's seeded, clustered synthetic store.

Every indexer is built the way a user builds it: prepare() on the store's blocks, then indexing.  k-means is
deterministic, so all three get the same centroids (checked) and the lists are the same; only the stored rows differ.
Per nprobe, the three indexers' stage 1 (coarse search + list scan + de-duplication), stage 2 (max-sim of the candidates) and end-to-end
search are timed alternated in one run (CUDA-event medians after warm-up), with the bytes each stage reads over its
time and recall@top_n against the exact indexer.  Synthetic recall says nothing about real ColBERT embeddings.

    python scripts/bench_colbert_residual.py --out-dir DIR
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_colbert_e2e import power_limit_w, summary, timed  # noqa: E402
from matchmaker_b200 import interaction  # noqa: E402
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer, ColBERTResidualIndexer  # noqa: E402

N_DIRECTIONS = 16384


def run_point(args, dim, passages, nprobes, dev, g):
    lengths = torch.clamp(torch.round(torch.randn(passages, generator=g, device=dev) * 30 + 75), 10, 180).long()
    off = torch.zeros(passages + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lengths, 0)
    n_rows = int(off[-1])
    dirs = torch.nn.functional.normalize(torch.randn(N_DIRECTIONS, dim, generator=g, device=dev), dim=1)

    def around(n):
        x = dirs[torch.randint(0, N_DIRECTIONS, (n,), generator=g, device=dev)]
        return (x + 0.5 * torch.randn(n, dim, generator=g, device=dev) / dim ** 0.5).half()

    store = torch.cat([around(min(1 << 22, n_rows - a)) for a in range(0, n_rows, 1 << 22)])
    q = around(args.queries * args.lq).view(args.queries, args.lq, dim)
    off_np = off.cpu().numpy()
    cfg = {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": args.nlist,
           "faiss_ivf_search_probe_count": nprobes[0]}
    exact = ColBERTEndToEndIndexer(cfg, device=dev)
    exact.index_device(store, off_np)
    ivf = ColBERTIVFIndexer(cfg, device=dev)
    blocks = [store[a:a + (1 << 22)].cpu().numpy() for a in range(0, n_rows, 1 << 22)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ivf.prepare(blocks)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    ivf.index_device(exact.store, off_np)   # shares the exact indexer's rows
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    point = {"dim": dim, "passages": passages, "rows": n_rows,
             "build_s": {"kmeans": t1 - t0, "ivf_assign_layout": t2 - t1},
             "device_bytes_per_row": {"ivf": dim * 2 + 8 + 8}, "runs": {}}
    idx = {"ivf": ivf}
    for bits in (1, 2):
        r = ColBERTResidualIndexer({**cfg, "colbert_residual_bits": bits}, device=dev)
        torch.cuda.synchronize()
        a = time.perf_counter()
        r.prepare(blocks)   # k-means, then the bases and level tables
        torch.cuda.synchronize()
        b = time.perf_counter()
        r.index_device(store, off_np)
        torch.cuda.synchronize()
        c = time.perf_counter()
        point["build_s"][f"r{bits}"] = {"prepare": b - a, "assign_encode_layout": c - b}
        point["device_bytes_per_row"][f"r{bits}"] = dim * bits // 8 + 4 + 8 + 8
        point[f"r{bits}_same_centroids"] = bool(torch.equal(r.ivf.centroids, ivf.ivf.centroids))
        idx[f"r{bits}"] = r
    del blocks, store
    nq, lq, kp = args.queries, args.lq, args.token_top_k
    c = min(lq * kp, 4096)
    _, i_ex = exact.search_device(q, args.top_n, token_top_k=kp)
    for nprobe in nprobes:
        for x in idx.values():
            x.ivf.nprobe = nprobe
        toks = q.reshape(nq * lq, dim)
        probes = ivf.ivf.coarse(toks)
        pc = torch.bincount(probes[probes >= 0].view(-1), minlength=args.nlist)
        scan_rows = int((((pc + 127) // 128) * (ivf.list_offsets[1:] - ivf.list_offsets[:-1])).sum())
        t = {f"{k}_{s}": [] for k in idx for s in ("stage1", "stage2", "e2e")}
        cands, stage2 = {}, {}
        for k, x in idx.items():
            cands[k] = x.candidates_device(q, kp)[1]
            cand = cands[k]
            pair_d = torch.where(cand >= 0, cand, torch.full_like(cand, -1))
            pair_q = torch.arange(nq, device=dev, dtype=torch.int32).repeat_interleave(c)
            if k == "ivf":
                stage2[k] = (lambda x=x, pq=pair_q, pd=pair_d: interaction.maxsim_store(
                    q, x.store, x.offsets, pq, pd, x.max_doc_len))
            else:
                stage2[k] = (lambda x=x, pq=pair_q, pd=pair_d: interaction.maxsim_store_residual(
                    q, x.store, x.list_ids, x.base, x.weight, x.bits, x.offsets, pq, pd, x.max_doc_len))
        for _ in range(args.warmup):
            for k, x in idx.items():
                x.candidates_device(q, kp), stage2[k](), x.search_device(q, args.top_n, token_top_k=kp)
        for _ in range(args.reps):   # alternated in one run
            for k, x in idx.items():
                t[f"{k}_stage1"] += timed(lambda x=x: x.candidates_device(q, kp), 1, 0)
                t[f"{k}_stage2"] += timed(stage2[k], 1, 0)
                t[f"{k}_e2e"] += timed(lambda x=x: x.search_device(q, args.top_n, token_top_k=kp), 1, 0)
        run = {k: summary(v) for k, v in t.items()}
        cand_rows = int(sum(int(lengths[cands["ivf"][a][cands["ivf"][a] >= 0]].sum()) for a in range(nq)))
        for k, x in idx.items():
            row_b = dim * 2 if k == "ivf" else dim * x.bits // 8
            s1, s2 = statistics.median(t[f"{k}_stage1"]), statistics.median(t[f"{k}_stage2"])
            _, got = x.search_device(q, args.top_n, token_top_k=kp)
            recall = sum(len(set(got[a].tolist()) & set(v for v in i_ex[a].tolist() if v >= 0)) /
                         max(1, int((i_ex[a] >= 0).sum())) for a in range(nq)) / nq
            run[k] = {"stage1_ms": 1e3 * s1, "stage2_ms": 1e3 * s2, "queries_per_s": nq / statistics.median(t[f"{k}_e2e"]),
                      "stage1_scan_bytes": scan_rows * row_b, "stage1_scan_gb_per_s": scan_rows * row_b / s1 / 1e9,
                      "stage2_bytes": cand_rows * (row_b + (0 if k == "ivf" else 4)),
                      "stage2_gb_per_s": cand_rows * (row_b + (0 if k == "ivf" else 4)) / s2 / 1e9,
                      f"recall_at_{args.top_n}": recall}
        point["runs"][f"p{nprobe}"] = run
        print(json.dumps({f"dim{dim}_p{nprobe}": {k: run[k] for k in idx}}), flush=True)
    return point


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=250_000)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--lq", type=int, default=32)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nprobe", type=int, nargs="+", default=[4, 16, 64])
    ap.add_argument("--token-top-k", type=int, default=64)
    ap.add_argument("--top-n", type=int, default=1000)
    ap.add_argument("--dim768-passages", type=int, default=50_000, help="passages of the dim-768 point (0: skip)")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev).manual_seed(args.seed)
    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "queries": args.queries,
           "lq": args.lq, "top_n": args.top_n, "nlist": args.nlist, "token_top_k": args.token_top_k, "points": []}
    res["points"].append(run_point(args, args.dim, args.passages, args.nprobe, dev, g))
    torch.cuda.empty_cache()
    if args.dim768_passages:
        res["points"].append(run_point(args, 768, args.dim768_passages, [16], dev, g))
    print(json.dumps(res))
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, "bench_colbert_residual.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
