"""TK re-ranking over an encoded document store on one GPU, against the paths it replaces.

Shape: BASELINE config 2's TK interaction (Lq 30, D 300, 11 or 21 kernels) with MSMARCO-shaped passage lengths
(live rows drawn around 60, 5 to 200, padded length 200), --queries queries of --cands candidates each from a pool of
--docs passages.  Four paths on the same pairs:

- store: ``interaction.kernel_pool_store`` alone (the store mode of the kernel-pooling kernel);
- padded: ``interaction.kernel_pool`` on the same passages gathered into [pairs, 200, D] with masks (the gather is
  made beforehand and not timed);
- forward: ``ECAI20_TK.forward`` on the raw embeddings of the pairs of one query (it runs the document transformer), per
  pair;
- rerank: ``TKDocumentStore.rerank`` end to end (pairs, kernel, top-k selection).

Times are CUDA-event medians over --rounds rounds, the paths alternated within each round after a warm-up.  Bytes per
pair = live_rows * D * 4 + 4 (the score) + the query's Lq * D * 4 over its candidates; the padded path's are the same
with 200 rows and the mask.  Fraction of the HBM bound = those bytes / 3.35 TB/s (H100 SXM data sheet) / time.

    python scripts/bench_tk_store.py --out-dir DIR
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

from bench_colbert_e2e import power_limit_w  # noqa: E402
from bench_kernel_pool_wide import sm_clock_mhz  # noqa: E402
from matchmaker_b200 import interaction  # noqa: E402
from matchmaker_b200.rankers.tk import ECAI20_TK  # noqa: E402
from matchmaker_b200.retrieval import TKDocumentStore  # noqa: E402
from oracle import interaction_oracle as O  # noqa: E402

HBM_PEAK_BPS = 3.35e12   # H100 SXM data sheet
LQ, D, LD = 30, 300, 200


def timed(fn, rounds_times, key, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    rounds_times.setdefault(key, []).append(a.elapsed_time(b) / 1e3 / steps)


def run(args, K):
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(K)
    torch.manual_seed(K)
    mu, sigma = O.knrm_kernel_mus(K), O.knrm_kernel_sigmas(K)
    model = ECAI20_TK(D, mu, sigma, att_heads=10, att_layer=2, att_ff_dim=100, max_length=LD,
                      use_diff_posencoding=True, mix_hybrid_context=True).to(dev).eval()
    lens = torch.randn(args.docs, generator=g, device=dev).mul(25).add(60).round().clamp(5, LD).long()
    emb = torch.randn(args.docs, LD, D, generator=g, device=dev) * 0.5
    dmask = (torch.arange(LD, device=dev).unsqueeze(0) < lens.unsqueeze(1)).float()
    rows, off_parts = [], [torch.zeros(1, dtype=torch.int64, device=dev)]
    with torch.no_grad():
        for b0 in range(0, args.docs, 256):
            r, l = model.encode_documents(emb[b0:b0 + 256], dmask[b0:b0 + 256])
            rows.append(r)
            off_parts.append(l)
    store = torch.cat(rows)
    off = torch.cumsum(torch.cat(off_parts), 0)
    nq, C = args.queries, args.cands
    q = torch.randn(nq, LQ, D, generator=g, device=dev) * 0.5
    qm = (torch.arange(LQ, device=dev).unsqueeze(0) < torch.randint(5, LQ + 1, (nq, 1), generator=g, device=dev)).float()
    with torch.no_grad():
        qctx = model.forward_representation(q, qm, model.positional_features_q[:, :LQ, :])
    cand = torch.stack([torch.randperm(args.docs, generator=g, device=dev)[:C] for _ in range(nq)])
    pq = torch.arange(nq, device=dev, dtype=torch.int32).repeat_interleave(C)
    pd = cand.reshape(-1).to(torch.int32)
    w, alpha = model.kernel_bin_weights.weight.detach(), model.kernel_alpha_scaler.detach()
    mu_t, sg_t = model.mu, model.sigma
    max_len = int(lens.max())
    # padded gather of the same pairs
    n_pairs = pq.numel()
    pad = torch.zeros(n_pairs, LD, D, device=dev)
    pmask = torch.zeros(n_pairs, LD, device=dev)
    plen = lens[pd.long()]
    for p0 in range(0, n_pairs, 1000):
        for j, di in enumerate(pd[p0:p0 + 1000].tolist()):
            a, b = int(off[di]), int(off[di + 1])
            pad[p0 + j, :b - a] = store[a:b]
            pmask[p0 + j, :b - a] = 1
    qg = qctx[pq.long()].contiguous()
    qmg = qm[pq.long()].contiguous()
    cfg = {"token_dim": D, "faiss_use_gpu": True, "token_dtype": "float32"}
    st = TKDocumentStore(cfg, model)
    local = (off - off[0]).cpu().numpy()
    st._set(local, 0, args.docs, store, None)
    # one query's pairs through the full forward
    fq, fd = q[:1].expand(C, -1, -1).contiguous(), emb[cand[0]]
    fqm, fdm = qm[:1].expand(C, -1).contiguous(), dmask[cand[0]]

    with torch.no_grad():
        s_store = interaction.kernel_pool_store(qctx, qm, store, off, pq, pd, mu_t, sg_t, w, alpha, max_doc_len=max_len)
        s_pad = interaction.kernel_pool(qg, pad, qmg, pmask, mu_t, sg_t, w, alpha)["score"]
        s_fwd = model(fq, fd, fqm, fdm)
    max_rel_store_vs_pad = float(((s_store - s_pad).abs() / s_pad.abs().clamp(min=1e-6)).max())
    max_rel_store_vs_fwd = float(((s_store[:C] - s_fwd).abs() / s_fwd.abs().clamp(min=1e-6)).max())

    paths = {
        "store": lambda: interaction.kernel_pool_store(qctx, qm, store, off, pq, pd, mu_t, sg_t, w, alpha,
                                                       max_doc_len=max_len),
        "padded": lambda: interaction.kernel_pool(qg, pad, qmg, pmask, mu_t, sg_t, w, alpha),
        "forward": lambda: model(fq, fd, fqm, fdm),
        "rerank": lambda: st.rerank(qctx, qm, cand, top_n=100),
    }
    pairs = {"store": n_pairs, "padded": n_pairs, "forward": C, "rerank": n_pairs}
    times = {}
    with torch.no_grad():
        for fn in paths.values():   # warm-up
            fn()
        torch.cuda.synchronize()
        for r in range(args.rounds):
            order = list(paths) if r % 2 == 0 else list(reversed(paths))
            for k in order:
                timed(paths[k], times, k, args.steps if k != "forward" else max(1, args.steps // 10))
    live = float(plen.float().mean())
    q_amort = LQ * D * 4 / C
    bytes_store = live * D * 4 + 4 + q_amort
    bytes_pad = LD * D * 4 + LD * 4 + 4 + q_amort
    out = {"K": K, "queries": nq, "cands": C, "docs": args.docs, "mean_live_rows": live, "max_doc_len": max_len,
           "store_rows": int(store.shape[0]), "store_bytes": int(store.numel() * 4),
           "bytes_per_pair_store": bytes_store, "bytes_per_pair_padded": bytes_pad,
           "max_rel_diff_store_vs_padded": max_rel_store_vs_pad, "max_rel_diff_store_vs_forward": max_rel_store_vs_fwd}
    for k, ts in times.items():
        t = statistics.median(ts)
        out[k] = {"s_per_call": t, "pairs_per_s": pairs[k] / t, "spread": [min(ts), max(ts)]}
    for k, b in (("store", bytes_store), ("padded", bytes_pad), ("rerank", bytes_store)):
        out[k]["hbm_fraction"] = pairs[k] * b / HBM_PEAK_BPS / out[k]["s_per_call"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=tempfile.gettempdir())
    ap.add_argument("--queries", type=int, default=16)
    ap.add_argument("--cands", type=int, default=1000)
    ap.add_argument("--docs", type=int, default=20000)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tk_store: no GPU")
    res = {"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit_w(), "sm_clock_max_mhz": sm_clock_mhz(),
           "results": [run(args, K) for K in (11, 21)]}
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "bench_tk_store.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
