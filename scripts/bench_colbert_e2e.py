"""ColBERT end-to-end retrieval benchmark (one GPU): per-stage times of ColBERTEndToEndIndexer.search_device over a
seeded synthetic token store, and an alternated A/B of stage 2 (store-mode max-sim) against the padded tensor-core
max-sim on the same candidate pairs.

Store: passage lengths clip(N(75, 30), 10, 180) (BASELINE config 3), dim 128, fp16, generated on the GPU.
Queries: 64 x Lq 32.  k' in {64, 256}, top_n 1000.  Times are CUDA-event medians after warm-up.

    python scripts/bench_colbert_e2e.py --passages 1000000 --out-dir DIR
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from matchmaker_b200 import interaction  # noqa: E402
from matchmaker_b200.retrieval import ColBERTEndToEndIndexer  # noqa: E402

H100_SXM_HBM_BPS = 3.35e12   # data-sheet HBM3 bandwidth of the H100 SXM


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) * 1e-3)
    return ts


def summary(ts):
    return {"median_s": statistics.median(ts), "min_s": min(ts), "max_s": max(ts), "n": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passages", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=64)
    ap.add_argument("--lq", type=int, default=32)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--top-n", type=int, default=1000)
    ap.add_argument("--token-top-k", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ab-rounds", type=int, default=20)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()

    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator(device=dev).manual_seed(args.seed)
    lengths = torch.clamp(torch.round(torch.randn(args.passages, generator=g, device=dev) * 30 + 75), 10, 180).long()
    off = torch.zeros(args.passages + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(lengths, 0)
    n_rows = int(off[-1])
    store = (torch.randn(n_rows, args.dim, generator=g, device=dev, dtype=torch.float16) * 0.1)
    q = (torch.randn(args.queries, args.lq, args.dim, generator=g, device=dev, dtype=torch.float16) * 0.1)
    idx = ColBERTEndToEndIndexer({"token_dim": args.dim, "faiss_use_gpu": True, "token_dtype": "float16"}, device=dev)
    idx.index_device(store, off.cpu().numpy())
    del store
    torch.cuda.synchronize()

    res = {"card": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "passages": args.passages,
           "rows": n_rows, "dim": args.dim, "queries": args.queries, "lq": args.lq, "top_n": args.top_n,
           "store_gb": n_rows * args.dim * 2 / 1e9, "runs": {}}
    nq, lq = args.queries, args.lq
    for kp in args.token_top_k:
        toks = q.reshape(nq * lq, args.dim)
        c = min(lq * kp, 4096)
        st = {}
        st["stage1"] = timed(lambda: interaction.flat_ip_topk(toks, idx.tokens.flat, kp, ids=idx.row_ids), args.reps, args.warmup)
        hs, hi = interaction.flat_ip_topk(toks, idx.tokens.flat, kp, ids=idx.row_ids)
        st["unique"] = timed(lambda: interaction.topk_unique(hs.view(nq, lq * kp), hi.view(nq, lq * kp), c),
                             args.reps, args.warmup)
        _, cand = interaction.topk_unique(hs.view(nq, lq * kp), hi.view(nq, lq * kp), c)
        pair_d = torch.where(cand >= 0, cand, torch.full_like(cand, -1))
        pair_q = torch.arange(nq, device=dev, dtype=torch.int32).repeat_interleave(c)
        st["stage2"] = timed(lambda: interaction.maxsim_store(q, idx.store, idx.offsets, pair_q, pair_d, idx.max_doc_len),
                             args.reps, args.warmup)
        scores = interaction.maxsim_store(q, idx.store, idx.offsets, pair_q, pair_d, idx.max_doc_len).view(nq, c)
        st["merge"] = timed(lambda: interaction.topk_merge(scores, cand, args.top_n), args.reps, args.warmup)
        st["end_to_end"] = timed(lambda: idx.search_device(q, args.top_n, token_top_k=kp), args.reps, args.warmup)
        valid = cand >= 0
        cand_len = (idx.offsets[1:] - idx.offsets[:-1])[cand.clamp(min=0)] * valid
        n_pairs = int(valid.sum())
        bytes2 = int(cand_len.sum()) * args.dim * 2
        s1, s2 = statistics.median(st["stage1"]), statistics.median(st["stage2"])
        run = {k: summary(v) for k, v in st.items()}
        run.update({"candidates_per_query": c, "valid_pairs": n_pairs,
                    "stage1_tflops": 2 * args.dim * nq * lq * n_rows / s1 / 1e12,
                    "stage2_pairs_per_s": n_pairs / s2, "stage2_bytes_per_s": bytes2 / s2,
                    "stage2_hbm_share": bytes2 / s2 / H100_SXM_HBM_BPS,
                    "queries_per_s": nq / statistics.median(st["end_to_end"])})
        res["runs"][f"k{kp}"] = run
        print(json.dumps({f"k{kp}": {k: (v["median_s"] if isinstance(v, dict) else v) for k, v in run.items()}}), flush=True)

    # A/B of stage 2: the same candidate pairs (k' = first value) scored from the store and from the padded layout
    kp = args.token_top_k[0]
    c = min(lq * kp, 4096)
    toks = q.reshape(nq * lq, args.dim)
    hs, hi = interaction.flat_ip_topk(toks, idx.tokens.flat, kp, ids=idx.row_ids)
    _, cand = interaction.topk_unique(hs.view(nq, lq * kp), hi.view(nq, lq * kp), c)
    keep = (cand >= 0).reshape(-1)
    pair_d = cand.reshape(-1)[keep]
    pair_q = torch.arange(nq, device=dev, dtype=torch.int32).repeat_interleave(c)[keep]
    L = idx.max_doc_len
    lens = (idx.offsets[1:] - idx.offsets[:-1])[pair_d]
    pos = torch.arange(L, device=dev)
    mask = pos.unsqueeze(0) < lens.unsqueeze(1)                                    # [P, L]
    rows = (idx.offsets[pair_d].unsqueeze(1) + pos.unsqueeze(0)).clamp(max=idx.store.shape[0] - 1)
    padded = idx.store[rows] * mask.unsqueeze(-1).to(idx.store.dtype)               # [P, L, dim], pair p = doc p
    pd_pad = torch.arange(pair_d.numel(), device=dev, dtype=torch.int32)
    pd_store = pair_d.to(torch.int32)
    f_store = lambda: interaction.maxsim_store(q, idx.store, idx.offsets, pair_q, pd_store, L)  # noqa: E731
    f_pad = lambda: interaction.maxsim(q, padded, None, mask, pair_q=pair_q, pair_d=pd_pad, impl="tcgen05")  # noqa: E731
    same = torch.equal(f_store(), f_pad())
    for f in (f_store, f_pad):
        timed(f, 0, args.warmup)
    ts_store, ts_pad = [], []
    for r in range(args.ab_rounds):
        order = [(f_store, ts_store), (f_pad, ts_pad)] if r % 2 == 0 else [(f_pad, ts_pad), (f_store, ts_store)]
        for f, acc in order:
            acc += timed(f, 1, 0)
    ms, mp = statistics.median(ts_store), statistics.median(ts_pad)
    res["stage2_ab"] = {"pairs": int(pair_d.numel()), "padded_len": L, "bit_identical": same,
                        "store": summary(ts_store), "padded_tcgen05": summary(ts_pad), "store_speedup": mp / ms}
    print(json.dumps({"stage2_ab": {"store_s": ms, "padded_s": mp, "speedup": mp / ms, "bit_identical": same}}), flush=True)
    del padded, mask, rows

    out_dir = args.out_dir or tempfile.mkdtemp(prefix="colbert_e2e_bench_")
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, f"colbert_e2e_{time.strftime('%Y%m%d_%H%M%S')}.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"], "power_limit_w": res["power_limit_w"], "json": path}))


if __name__ == "__main__":
    main()
