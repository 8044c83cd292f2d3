"""ColBERT retrieval with the inverted-file token index (retrieval.ColBERTIVFIndexer) against the exact indexer on one
GPU, over the same seeded, clustered synthetic token store.

Store: passage lengths clip(N(75, 30), 10, 180) as in bench_colbert_e2e.py, dim 128, fp16, rows drawn around 16 384
random unit directions (so that an inverted file and recall mean something), generated on the GPU.  Queries: 64 x Lq
32 drawn the same way.  Reports the build split (k-means, assignment, layout), stage-1 times of both indexers
alternated in one run, the other stages, end-to-end queries/s, recall@top_n against the exact indexer, the bytes the
gather scan reads over its time, and an A/B of the gather scan against ivf_search over a list-ordered copy of the same
rows (alternated, checked bit-identical).  Times are CUDA-event medians after warm-up.

    python scripts/bench_colbert_ivf.py --passages 250000 --out-dir DIR
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
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer  # noqa: E402

N_DIRECTIONS = 16384


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=250_000)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--lq", type=int, default=32)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nprobe", type=int, nargs="+", default=[4, 16, 64])
    ap.add_argument("--token-top-k", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--top-n", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()

    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev).manual_seed(args.seed)
    lengths = torch.clamp(torch.round(torch.randn(args.passages, generator=g, device=dev) * 30 + 75), 10, 180).long()
    off = torch.zeros(args.passages + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lengths, 0)
    n_rows, dim = int(off[-1]), args.dim
    dirs = torch.nn.functional.normalize(torch.randn(N_DIRECTIONS, dim, generator=g, device=dev), dim=1)

    def around(n):
        x = dirs[torch.randint(0, N_DIRECTIONS, (n,), generator=g, device=dev)]
        return (x + 0.5 * torch.randn(n, dim, generator=g, device=dev) / dim ** 0.5).half()

    store = torch.cat([around(min(1 << 22, n_rows - a)) for a in range(0, n_rows, 1 << 22)])
    q = around(args.queries * args.lq).view(args.queries, args.lq, dim)
    off_np = off.cpu().numpy()
    cfg = {"token_dim": dim, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": args.nlist,
           "faiss_ivf_search_probe_count": args.nprobe[0]}
    exact = ColBERTEndToEndIndexer(cfg, device=dev)
    exact.index_device(store, off_np)
    ivf = ColBERTIVFIndexer(cfg, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ivf.prepare([store[a:a + (1 << 22)].cpu().numpy() for a in range(0, n_rows, 1 << 22)])   # IVFIndexer's k-means
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    # index_device(exact.store) shares the exact indexer's rows: both indexers read the same HBM copy
    ivf.index_device(exact.store, off_np)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    del store
    lens = (ivf.list_offsets[1:] - ivf.list_offsets[:-1]).float()
    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "passages": args.passages,
           "rows": n_rows, "dim": dim, "queries": args.queries, "lq": args.lq, "top_n": args.top_n, "nlist": args.nlist,
           "build_s": {"kmeans": t1 - t0, "assign_layout": t2 - t1},
           "list_len": {"mean": float(lens.mean()), "max": int(lens.max()), "empty": int((lens == 0).sum())},
           "runs": {}}
    nq, lq = args.queries, args.lq
    toks = q.reshape(nq * lq, dim)
    for kp in args.token_top_k:
        c = min(lq * kp, 4096)
        s_ex, i_ex = exact.search_device(q, args.top_n, token_top_k=kp)
        for nprobe in args.nprobe:
            ivf.ivf.nprobe = nprobe
            probes = ivf.ivf.coarse(toks)

            def gather():
                return interaction.ivf_search(toks, ivf.tokens.flat, ivf.row_ids, ivf.list_offsets, probes, kp,
                                              ivf.max_list_len, row_index=ivf.row_index)
            st = {"stage1_exact": [], "stage1_ivf": []}
            for _ in range(args.warmup):
                interaction.flat_ip_topk(toks, exact.tokens.flat, kp, ids=exact.row_ids)
                ivf.candidates_device(q, kp)
            for _ in range(args.reps):   # alternated in one run
                st["stage1_exact"] += timed(lambda: interaction.flat_ip_topk(toks, exact.tokens.flat, kp, ids=exact.row_ids), 1, 0)
                st["stage1_ivf"] += timed(lambda: (ivf.ivf.coarse(toks), gather()), 1, 0)
            st["coarse"] = timed(lambda: ivf.ivf.coarse(toks), args.reps, args.warmup)
            st["gather_scan"] = timed(gather, args.reps, args.warmup)
            hs, hi = gather()
            st["unique"] = timed(lambda: interaction.topk_unique(hs.view(nq, lq * kp), hi.view(nq, lq * kp), c),
                                 args.reps, args.warmup)
            st["end_to_end"] = timed(lambda: ivf.search_device(q, args.top_n, token_top_k=kp), args.reps, args.warmup)
            s, i = ivf.search_device(q, args.top_n, token_top_k=kp)
            recall = sum(len(set(i[a].tolist()) & set(x for x in i_ex[a].tolist() if x >= 0)) /
                         max(1, int((i_ex[a] >= 0).sum())) for a in range(nq)) / nq
            # rows the gather scan reads: every (live token, probed list) pair reads its list once per 128-token chunk;
            # counted as one read per distinct (list, chunk) item
            pc = torch.bincount(probes[probes >= 0].view(-1), minlength=args.nlist)
            chunks = (pc + 127) // 128
            scan_bytes = int((chunks * (ivf.list_offsets[1:] - ivf.list_offsets[:-1])).sum()) * dim * 2
            run = {k: summary(v) for k, v in st.items()}
            run.update({"recall_at_top_n": recall, "scan_bytes": scan_bytes,
                        "scan_bytes_per_s": scan_bytes / statistics.median(st["gather_scan"]),
                        "stage1_speedup": statistics.median(st["stage1_exact"]) / statistics.median(st["stage1_ivf"]),
                        "queries_per_s": nq / statistics.median(st["end_to_end"])})
            if kp == args.token_top_k[0]:   # A/B: gather against a materialised list-ordered copy of the same rows
                rows_c, ids_c = ivf.tokens.flat[ivf.row_index].contiguous(), ivf.row_ids[ivf.row_index].contiguous()

                def copy():
                    return interaction.ivf_search(toks, rows_c, ids_c, ivf.list_offsets, probes, kp, ivf.max_list_len)
                cs, ci = copy()
                ab = {"gather": [], "copy": []}
                for _ in range(args.reps):
                    ab["gather"] += timed(gather, 1, 0)
                    ab["copy"] += timed(copy, 1, 0)
                run["ab_gather_vs_copy"] = {"gather": summary(ab["gather"]), "copy": summary(ab["copy"]),
                                            "bit_identical": bool(torch.equal(cs.view(torch.int32), hs.view(torch.int32))
                                                                  and torch.equal(ci, hi))}
                del rows_c, ids_c
            res["runs"][f"k{kp}_p{nprobe}"] = run
            print(json.dumps({f"k{kp}_p{nprobe}": {"recall": recall, "stage1_ivf_ms": 1e3 * statistics.median(st["stage1_ivf"]),
                                                   "stage1_exact_ms": 1e3 * statistics.median(st["stage1_exact"])}}), flush=True)
    print(json.dumps(res))
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, "bench_colbert_ivf.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
