"""ColBERT retrieval over the E4M3 token store (``colbert_store_dtype: "float8_e4m3"``, DESIGN 3.4i) against the fp16
store on one GPU, exact (ColBERTEndToEndIndexer) and IVF (ColBERTIVFIndexer), over bench_colbert_residual.py's seeded,
clustered synthetic store at dim 128 and dim 768.

The fp8 IVF indexer takes the fp16 one's centroids, so both have the same lists.  Per point, every indexer's stage 1
(token search + de-duplication), stage 2 (max-sim of its candidates) and end-to-end search are timed alternated in one
run (CUDA-event medians after warm-up), with the bytes each stage reads over its time and recall@top_n against the fp16
exact indexer.  Synthetic recall says nothing about real ColBERT embeddings.

    python scripts/bench_colbert_fp8.py --out-dir DIR
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_colbert_e2e import power_limit_w, summary, timed  # noqa: E402
from matchmaker_b200 import interaction  # noqa: E402
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer  # noqa: E402

N_DIRECTIONS = 16384


def run_point(args, dim, passages, nprobe, dev, g):
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
           "faiss_ivf_search_probe_count": nprobe}
    fp8 = {**cfg, "colbert_store_dtype": "float8_e4m3"}
    idx = {"exact_fp16": ColBERTEndToEndIndexer(cfg, device=dev), "exact_fp8": ColBERTEndToEndIndexer(fp8, device=dev),
           "ivf_fp16": ColBERTIVFIndexer(cfg, device=dev), "ivf_fp8": ColBERTIVFIndexer(fp8, device=dev)}
    blocks = [store[a:a + (1 << 22)].cpu().numpy() for a in range(0, n_rows, 1 << 22)]
    idx["ivf_fp16"].prepare(blocks)
    idx["ivf_fp8"].ivf.set_centroids(idx["ivf_fp16"].ivf.centroids)
    del blocks
    for x in idx.values():
        x.index_device(store, off_np)
    point = {"dim": dim, "passages": passages, "rows": n_rows, "nprobe": nprobe, "store_scale": idx["exact_fp8"].store_scale,
             "same_layout": bool(torch.equal(idx["ivf_fp16"].row_index, idx["ivf_fp8"].row_index)),
             "store_bytes_per_row": {"fp16": dim * 2 + 8, "fp8": dim + 8}}
    del store
    nq, lq, kp = args.queries, args.lq, args.token_top_k
    c = min(lq * kp, 4096)
    _, i_ref = idx["exact_fp16"].search_device(q, args.top_n, token_top_k=kp)
    t = {f"{k}_{s}": [] for k in idx for s in ("stage1", "stage2", "e2e")}
    cands, stage2 = {}, {}
    for k, x in idx.items():
        qs = x.tokens.queries(q)[0]
        cands[k] = x.candidates_device(q, kp, qs)[1]
        pair_d = cands[k]
        pair_q = torch.arange(nq, device=dev, dtype=torch.int32).repeat_interleave(c)
        stage2[k] = (lambda x=x, qs=qs, pq=pair_q, pd=pair_d: interaction.maxsim_store(
            qs, x.store, x.offsets, pq, pd, x.max_doc_len))
    for _ in range(args.warmup):
        for k, x in idx.items():
            x.candidates_device(q, kp), stage2[k](), x.search_device(q, args.top_n, token_top_k=kp)
    for _ in range(args.reps):   # alternated in one run
        for k, x in idx.items():
            t[f"{k}_stage1"] += timed(lambda x=x: x.candidates_device(q, kp), 1, 0)
            t[f"{k}_stage2"] += timed(stage2[k], 1, 0)
            t[f"{k}_e2e"] += timed(lambda x=x: x.search_device(q, args.top_n, token_top_k=kp), 1, 0)
    run = {k: summary(v) for k, v in t.items()}
    ivf = idx["ivf_fp16"]
    probes = ivf.ivf.coarse(q.reshape(nq * lq, dim))
    pc = torch.bincount(probes[probes >= 0].view(-1), minlength=args.nlist)
    ivf_rows = int((((pc + 127) // 128) * (ivf.list_offsets[1:] - ivf.list_offsets[:-1])).sum())
    exact_rows = ((nq * lq + 127) // 128) * n_rows     # every block of 128 query tokens reads every row
    for k, x in idx.items():
        row_b = dim if k.endswith("fp8") else dim * 2
        scan_rows = ivf_rows if k.startswith("ivf") else exact_rows
        cand_rows = int(sum(int(lengths[cands[k][a][cands[k][a] >= 0]].sum()) for a in range(nq)))
        s1, s2 = statistics.median(t[f"{k}_stage1"]), statistics.median(t[f"{k}_stage2"])
        _, got = x.search_device(q, args.top_n, token_top_k=kp)
        recall = sum(len(set(got[a].tolist()) & set(v for v in i_ref[a].tolist() if v >= 0)) /
                     max(1, int((i_ref[a] >= 0).sum())) for a in range(nq)) / nq
        run[k] = {"stage1_ms": 1e3 * s1, "stage2_ms": 1e3 * s2, "queries_per_s": nq / statistics.median(t[f"{k}_e2e"]),
                  "stage1_scan_bytes": scan_rows * row_b, "stage1_scan_gb_per_s": scan_rows * row_b / s1 / 1e9,
                  "stage2_bytes": cand_rows * row_b, "stage2_gb_per_s": cand_rows * row_b / s2 / 1e9,
                  f"recall_at_{args.top_n}": recall}
    point["runs"] = run
    print(json.dumps({f"dim{dim}": {k: run[k] for k in idx}}), flush=True)
    return point


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=100_000)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--lq", type=int, default=32)
    ap.add_argument("--nlist", type=int, default=1024)
    ap.add_argument("--nprobe", type=int, default=16)
    ap.add_argument("--token-top-k", type=int, default=64)
    ap.add_argument("--top-n", type=int, default=1000)
    ap.add_argument("--dim768-passages", type=int, default=20_000, help="passages of the dim-768 point (0: skip)")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev).manual_seed(args.seed)
    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "queries": args.queries,
           "lq": args.lq, "top_n": args.top_n, "nlist": args.nlist, "token_top_k": args.token_top_k, "points": []}
    res["points"].append(run_point(args, 128, args.passages, args.nprobe, dev, g))
    torch.cuda.empty_cache()
    if args.dim768_passages:
        res["points"].append(run_point(args, 768, args.dim768_passages, args.nprobe, dev, g))
    print(json.dumps(res))
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, "bench_colbert_fp8.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
