"""PLAID centroid-interaction search (``colbert_plaid_ndocs``, retrieval.colbert_plaid) against the token-scan IVF
search of ColBERTIVFIndexer and ColBERTResidualIndexer (b = 2) on one GPU, over bench_colbert_residual.py's seeded,
clustered synthetic store (250 k passages, ~18.8 M rows, dim 128) with rows and queries unit-normalised as ColBERT's.

Per nlist, one k-means (``prepare``) gives the centroids and the layout; the PLAID indexer loads that layout from a
file in a temporary directory and indexes the same device rows, so all indexers share centroids and lists; the
residual indexer trains the same centroids again (checked).  Per (nprobe, t_cs, ndocs, top_n):
- device time of each PLAID stage (CUDA-event medians): S + probes, candidates, pruned CI + select, full CI + select,
  exact max-sim + select (one rank: no cross-rank merge);
- candidates per query (mean, max) and the static candidate width;
- end-to-end queries/s of PLAID, and per nprobe of the two token-scan indexers (token_top_k 64), timed alternated;
- recall@10/100/1000 against ColBERTEndToEndIndexer (token_top_k 64).  Synthetic recall says nothing about real
  ColBERT embeddings.

    python scripts/bench_colbert_plaid.py --out-dir DIR
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_colbert_e2e import power_limit_w, timed  # noqa: E402
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer, ColBERTResidualIndexer  # noqa: E402

N_DIRECTIONS = 16384
TOKEN_TOP_K = 64


def make_store(args, dev, g):
    dim = args.dim
    lengths = torch.clamp(torch.round(torch.randn(args.passages, generator=g, device=dev) * 30 + 75), 10, 180).long()
    off = torch.zeros(args.passages + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lengths, 0)
    dirs = torch.nn.functional.normalize(torch.randn(N_DIRECTIONS, dim, generator=g, device=dev), dim=1)

    def around(n):
        x = dirs[torch.randint(0, N_DIRECTIONS, (n,), generator=g, device=dev)]
        return torch.nn.functional.normalize(x + 0.5 * torch.randn(n, dim, generator=g, device=dev) / dim ** 0.5,
                                             dim=1).half()

    n_rows = int(off[-1])
    store = torch.cat([around(min(1 << 22, n_rows - a)) for a in range(0, n_rows, 1 << 22)])
    q = around(args.queries * args.lq).view(args.queries, args.lq, dim)
    return store, off.cpu().numpy(), q


def recall(got, ref, k):
    return sum(len(set(got[a, :k].tolist()) & set(ref[a, :k].tolist())) / k for a in range(got.shape[0])) / got.shape[0]


def med_ms(ts):
    return 1e3 * statistics.median(ts)


def stage_times(x, q, top_n, reps):
    """Device time of each PLAID stage of one batch (the benchmark's queries fit one batch)."""
    p = x.plaid
    nq, lq, _ = q.shape
    qs, _ = x.tokens.queries(q)
    s, keep, probes = p.centroid_scores(x, q)
    cand = p.candidates(x, probes, lq)
    _, c1 = p.interaction(x, s, keep, cand, lq, p.ndocs)
    _, c2 = p.interaction(x, s, None, c1, lq, p.ndocs // 4)
    n_cand = (cand >= 0).sum(1).float()
    return {"s_probes_ms": med_ms(timed(lambda: p.centroid_scores(x, q), reps, 1)),
            "candidates_ms": med_ms(timed(lambda: p.candidates(x, probes, lq), reps, 1)),
            "pruned_ci_select_ms": med_ms(timed(lambda: p.interaction(x, s, keep, cand, lq, p.ndocs), reps, 1)),
            "full_ci_select_ms": med_ms(timed(lambda: p.interaction(x, s, None, c1, lq, p.ndocs // 4), reps, 1)),
            "exact_maxsim_select_ms": med_ms(timed(lambda: p.exact(x, qs, c2, top_n), reps, 1)),
            "candidates_mean": float(n_cand.mean()), "candidates_max": int(n_cand.max()), "cap": int(cand.shape[1])}


def run_nlist(args, nlist, store, off, q, blocks, exact_ids, dev):
    cfg = {"token_dim": args.dim, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": nlist,
           "faiss_ivf_search_probe_count": args.nprobe[0]}
    ivf = ColBERTIVFIndexer(cfg, device=dev)
    ivf.prepare(blocks)
    ivf.index_device(store, off)
    res = ColBERTResidualIndexer({**cfg, "colbert_residual_bits": 2}, device=dev)
    res.prepare(blocks)
    res.index_device(store, off)
    plaid = ColBERTIVFIndexer({**cfg, "colbert_plaid_ndocs": 4096}, device=dev)
    with tempfile.TemporaryDirectory() as tmp:
        ivf.save(os.path.join(tmp, "layout"))
        plaid.load(os.path.join(tmp, "layout"))
    plaid.index_device(store, off)   # the saved layout over the same rows: no assignment
    out = {"nlist": nlist, "residual_same_centroids": bool(torch.equal(res.ivf.centroids, ivf.ivf.centroids)),
           "longest_passage_list": plaid.plaid.max_plist_len, "runs": []}
    nq = q.shape[0]
    for nprobe in args.nprobe:
        for x in (ivf, res, plaid):
            x.ivf.nprobe = nprobe
        base = {"ivf": lambda: ivf.search_device(q, 1000, token_top_k=TOKEN_TOP_K),
                "residual_b2": lambda: res.search_device(q, 1000, token_top_k=TOKEN_TOP_K)}
        for t_cs in args.t_cs:
            for ndocs, top_n in ((1024, 100), (4096, 100), (4096, 1000)):
                plaid.plaid.threshold, plaid.plaid.ndocs = t_cs, ndocs
                fns = dict(base, plaid=lambda: plaid.search_device(q, top_n))
                ts = {k: [] for k in fns}
                for fn in fns.values():
                    fn()
                torch.cuda.synchronize()
                for _ in range(args.reps):   # alternated
                    for k, fn in fns.items():
                        ts[k] += timed(fn, 1, 0)
                _, got = plaid.search_device(q, top_n)
                got = got.cpu()
                run = {"nprobe": nprobe, "t_cs": t_cs, "ndocs": ndocs, "top_n": top_n,
                       "queries_per_s": {k: nq / statistics.median(v) for k, v in ts.items()},
                       "recall": {f"at_{k}": recall(got, exact_ids, k) for k in (10, 100, 1000) if k <= top_n},
                       "stages": stage_times(plaid, q, top_n, args.reps)}
                if ndocs == 4096 and top_n == 1000 and t_cs == args.t_cs[0]:
                    for k in base:
                        _, bi = (ivf if k == "ivf" else res).search_device(q, 1000, token_top_k=TOKEN_TOP_K)
                        run["recall"][f"{k}_at_1000"] = recall(bi.cpu(), exact_ids, 1000)
                        run["recall"][f"{k}_at_100"] = recall(bi.cpu(), exact_ids, 100)
                out["runs"].append(run)
                print(json.dumps({"nlist": nlist, **run}), flush=True)
    del ivf, res, plaid
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=250_000)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--lq", type=int, default=32)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--nlist", type=int, nargs="+", default=[4096, 65536])
    ap.add_argument("--nprobe", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--t-cs", type=float, nargs="+", default=[0.4, 0.45, 0.5])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev).manual_seed(args.seed)
    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "queries": args.queries,
           "lq": args.lq, "passages": args.passages, "nlists": []}
    store, off, q = make_store(args, dev, g)
    res["rows"] = int(store.shape[0])
    blocks = [store[a:a + (1 << 22)].cpu().numpy() for a in range(0, store.shape[0], 1 << 22)]
    exact = ColBERTEndToEndIndexer({"token_dim": args.dim, "faiss_use_gpu": True, "token_dtype": "float16"}, device=dev)
    exact.index_device(store, off)
    exact_ids = exact.search_device(q, 1000, token_top_k=TOKEN_TOP_K)[1].cpu()
    for nlist in args.nlist:
        res["nlists"].append(run_nlist(args, nlist, exact.store, off, q, blocks, exact_ids, dev))
    print(json.dumps(res))
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        with open(os.path.join(args.out_dir, "bench_colbert_plaid.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
