"""TKL re-ranking over an encoded document store on one GPU, against the paths it replaces.

Shape: TKL with 11 kernels, D 300, Lq 30 (the reference's query position limit), ``max_doc_length`` 2000 (C = 50 chunk
slots, W = 986 windows), passages of 100 to 2000 tokens with a mean near 1100, --queries queries of --cands candidates
each from a pool of --docs passages.  Four paths on the same pairs, each window scores + top-3 windows:

- store: ``interaction.tkl_store_window_scores`` + ``tkl_top_hills`` (the store mode of the window-score kernels);
- padded: ``interaction.tkl_window_scores`` + ``tkl_top_hills`` on the same chunks gathered into the padded layout with
  ``q[pair_q]`` (the gather is made beforehand and not timed);
- forward: ``TKL_sigir20.forward`` on the raw embeddings of --fwd-pairs pairs of one query (it runs the transformer over
  every packed chunk), per pair;
- rerank: ``TKLDocumentStore.rerank`` end to end (pairs, kernels, top-k selection).

Times are CUDA-event medians over --rounds rounds, the paths alternated within each round after a warm-up.  Bytes per
pair = packed chunks * 40 * (D * 4 + 4) (rows and mask bytes) + W * 4 (the window scores, written and read back by the
selection) + the query's Lq * D * 4 over its candidates; the padded path reads the same chunk bytes.  Fraction of the
HBM bound = those bytes / 3.35 TB/s (H100 SXM data sheet) / time.

    python scripts/bench_tkl_store.py --out-dir DIR
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
from matchmaker_b200 import interaction, synthetic  # noqa: E402
from matchmaker_b200.rankers.tkl import TKL_sigir20  # noqa: E402
from matchmaker_b200.retrieval import TKLDocumentStore  # noqa: E402

HBM_PEAK_BPS = 3.35e12   # H100 SXM data sheet
K, LQ, D, MAXLEN = 11, 30, 300, 2000
MU = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]


def timed(fn, rounds_times, key, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    rounds_times.setdefault(key, []).append(a.elapsed_time(b) / 1e3 / steps)


def run(args, sat):
    dev = torch.device("cuda")
    torch.manual_seed(5)
    g = torch.Generator().manual_seed(5)
    model = TKL_sigir20(D, MU, [0.1] * K, 10, 2, 300, MAXLEN, True, True, sat).to(dev).eval()
    lens = synthetic.synth_lengths(args.docs, 1100.0, 500.0, 100, MAXLEN, g)
    chunks, cmask, slots, counts = [], [], [], []
    with torch.no_grad():
        for b0 in range(0, args.docs, 32):
            n = min(32, args.docs - b0)
            L = int(lens[b0:b0 + n].max())
            dm = (torch.arange(L).unsqueeze(0) < lens[b0:b0 + n].unsqueeze(1)).float().to(dev)
            emb = torch.randn(n, L, D, generator=g).to(dev) * 0.5 * dm.unsqueeze(-1)
            c, m, s, k = model.encode_documents(emb, dm)
            chunks.append(c), cmask.append(m.to(torch.uint8)), slots.append(s), counts.append(k)
    chunks, cmask, slots, counts = torch.cat(chunks), torch.cat(cmask), torch.cat(slots), torch.cat(counts)
    cfg = {"token_dim": D, "faiss_use_gpu": True, "token_dtype": "float32"}
    st = TKLDocumentStore(cfg, model)
    off = torch.zeros(args.docs + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(counts.cpu(), 0) * 40
    st._set(off.numpy(), 0, args.docs, chunks, cmask.cpu(), slots.cpu().to(torch.int32))
    C = st.C
    W = (C * 40 - 30) // 2 + 1
    nq, nc = args.queries, args.cands
    q = torch.randn(nq, LQ, D, generator=g).to(dev) * 0.5
    qm = (torch.arange(LQ).unsqueeze(0) < torch.randint(5, LQ + 1, (nq, 1), generator=g)).float().to(dev)
    with torch.no_grad():
        qctx = model.forward_representation(q, qm, model.positional_features_q[:, :LQ, :])[0]
    cand = torch.stack([torch.randperm(args.docs, generator=g)[:nc] for _ in range(nq)]).to(dev)
    pq = torch.arange(nq, device=dev, dtype=torch.int32).repeat_interleave(nc)
    pd = cand.reshape(-1).to(torch.int32)
    n_pairs = pq.numel()
    sp, red = model._saturation_params()
    sp, red = sp.detach(), None if red is None else red.detach()
    # padded gather of the same pairs
    ps = st.doc_slots[pd.long()]
    packed = (ps >= 0).reshape(-1)
    idx = ps.reshape(-1)[packed].long()
    pch, pcm = st.chunks[idx].contiguous(), st.chunk_mask[idx].contiguous()
    qg, qmg = qctx[pq.long()].contiguous(), qm[pq.long()].contiguous()
    # forward over the first --fwd-pairs pairs of query 0, documents padded to max_doc_length
    nf = min(args.fwd_pairs, nc)
    fl = lens[cand[0, :nf].cpu()]
    fdm = (torch.arange(MAXLEN).unsqueeze(0) < fl.unsqueeze(1)).float().to(dev)
    fd = torch.randn(nf, MAXLEN, D, generator=g).to(dev) * 0.5 * fdm.unsqueeze(-1)
    fq, fqm = q[:1].expand(nf, -1, -1).contiguous(), qm[:1].expand(nf, -1).contiguous()

    def store():
        ws = interaction.tkl_store_window_scores(qctx, qm, st.chunks, st.chunk_mask, st.doc_slots, pq, pd, model.mu,
                                                 model.sigma, model.dense.weight, sat, sp, red)
        return interaction.tkl_top_hills(ws, model.chunk_scoring)[0]

    def padded():
        ws = interaction.tkl_window_scores(qg, qmg, pch, pcm, packed, C, model.mu, model.sigma, model.dense.weight, sat,
                                           sp, red)
        return interaction.tkl_top_hills(ws, model.chunk_scoring)[0]

    with torch.no_grad():
        s_store, s_pad = store(), padded()
    identical = bool(torch.equal(s_store, s_pad))
    paths = {"store": store, "padded": padded, "forward": lambda: model(fq, fd, fqm, fdm),
             "rerank": lambda: st.rerank(qctx, qm, cand, top_n=100)}
    pairs = {"store": n_pairs, "padded": n_pairs, "forward": nf, "rerank": n_pairs}
    times = {}
    with torch.no_grad():
        for fn in paths.values():   # warm-up
            fn()
        torch.cuda.synchronize()
        for r in range(args.rounds):
            order = list(paths) if r % 2 == 0 else list(reversed(paths))
            for k in order:
                timed(paths[k], times, k, args.steps if k != "forward" else 1)
    chunks_per_pair = float(counts[pd.long()].float().mean())
    bytes_pair = chunks_per_pair * 40 * (D * 4 + 1) + 2 * W * 4 + LQ * D * 4 / nc
    out = {"saturation": sat, "queries": nq, "cands": nc, "docs": args.docs, "mean_doc_tokens": float(lens.float().mean()),
           "C": C, "W": W, "mean_chunks_per_pair": chunks_per_pair, "store_chunks": int(chunks.shape[0]),
           "store_bytes": int(chunks.numel() * 4 + cmask.numel()),
           "store_mb_per_1100_token_doc": 28 * 40 * D * 4 / 1e6, "bytes_per_pair": bytes_pair,
           "store_bit_identical_to_padded": identical}
    for k, ts in times.items():
        t = statistics.median(ts)
        out[k] = {"s_per_call": t, "pairs_per_s": pairs[k] / t, "spread": [min(ts), max(ts)]}
    for k in ("store", "padded", "rerank"):
        out[k]["hbm_fraction"] = pairs[k] * bytes_pair / HBM_PEAK_BPS / out[k]["s_per_call"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out-dir", default=tempfile.gettempdir())
    ap.add_argument("--queries", type=int, default=8)
    ap.add_argument("--cands", type=int, default=256)
    ap.add_argument("--docs", type=int, default=1000)
    ap.add_argument("--fwd-pairs", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tkl_store: no GPU")
    res = {"gpu": torch.cuda.get_device_name(), "power_limit_w": power_limit_w(), "sm_clock_max_mhz": sm_clock_mhz(),
           "results": [run(args, sat) for sat in ("embedding", "log")]}
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, "bench_tkl_store.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
