"""CPU restatement of PLAID centroid-interaction search (retrieval.colbert_plaid): the query x centroid score table and
its keep mask, the passage lists of a layout, the candidate union, the pruned / full centroid interaction and the whole
pipeline with an exact last stage.  Test infrastructure: plain torch in fp64 on the CPU, no library call.  On inputs
where every fp32 sum is exact and every score an fp16 number, the library must agree bit for bit."""
from __future__ import annotations

import math
from typing import List

import numpy as np
import torch

FLT_MAX = 3.4028234663852886e38


def lqp(lq: int) -> int:
    return 32 * ((lq + 31) // 32)


def live_tokens(q: torch.Tensor) -> torch.Tensor:
    """[Nq, Lq] bool: a token is live when one of its fp16 elements is nonzero."""
    return (q.to(torch.float16) != 0).any(-1)


def centroid_scores(q: torch.Tensor, cents: torch.Tensor, t_cs: float):
    """(S [Nq, nlist, LQP] fp64 holding fp16 values, 0 past Lq; keep [Nq, nlist] bool)."""
    nq, lq, _ = q.shape
    s = torch.einsum("qid,cd->qci", q.to(torch.float16).double(), cents.to(torch.float16).double())
    s = s.to(torch.float16).double()
    out = torch.zeros(nq, cents.shape[0], lqp(lq), dtype=torch.float64)
    out[:, :, :lq] = s
    live = live_tokens(q)
    keep = torch.zeros(nq, cents.shape[0], dtype=torch.bool)
    for a in range(nq):
        if live[a].any():
            keep[a] = s[a][:, live[a]].max(-1).values >= t_cs
    return out, keep


def keep_words(keep: torch.Tensor) -> torch.Tensor:
    """[Nq, nlist] bool -> [Nq, ceil(nlist / 32)] int32 bit words (bit c % 32 of word c / 32)."""
    nq, nlist = keep.shape
    w = (nlist + 31) // 32
    bits = np.zeros((nq, 32 * w), dtype=np.uint64)
    bits[:, :nlist] = keep.numpy()
    words = (bits.reshape(nq, w, 32) << np.arange(32, dtype=np.uint64)).sum(-1).astype(np.uint32)
    return torch.from_numpy(words.view(np.int32).copy())


def passage_lists(row_index: torch.Tensor, list_offsets: torch.Tensor, row_pid: torch.Tensor) -> List[List[int]]:
    """Per list, its rows' distinct passages in ascending order, by a plain loop."""
    out = []
    for l in range(list_offsets.numel() - 1):
        rows = row_index[int(list_offsets[l]):int(list_offsets[l + 1])].tolist()
        out.append(sorted(set(int(row_pid[r]) for r in rows)))
    return out


def flatten_lists(plists: List[List[int]]):
    """(plist_offsets, plist_pids) of per-list passage lists."""
    off = [0]
    for p in plists:
        off.append(off[-1] + len(p))
    return torch.tensor(off, dtype=torch.int64), torch.tensor([x for p in plists for x in p], dtype=torch.int32)


def candidates(probes: torch.Tensor, plists: List[List[int]], cap: int, first_doc: int = 0) -> torch.Tensor:
    """[Nq, cap] int64: the union of the probed lists' passages (probes outside [0, nlist) probe nothing), as
    first_doc + pid ascending, then -1."""
    out = torch.full((probes.shape[0], cap), -1, dtype=torch.int64)
    for a in range(probes.shape[0]):
        u = sorted(set(p for l in probes[a].tolist() if 0 <= l < len(plists) for p in plists[l]))[:cap]
        out[a, :len(u)] = torch.tensor(u, dtype=torch.int64) + first_doc
    return out


def interaction(s: torch.Tensor, keep, list_ids: torch.Tensor, offsets, cand: torch.Tensor, lq: int,
                first_doc: int = 0) -> torch.Tensor:
    """[Nq, C] fp64: sum over i < lq of the max over the passage's rows whose list is kept (keep None: every row) of
    S[q][list][i]; -inf when no row qualifies or the candidate is void (outside the rank's passages)."""
    off = torch.as_tensor(offsets, dtype=torch.int64)
    n_docs = off.numel() - 1
    out = torch.full(cand.shape, -math.inf, dtype=torch.float64)
    for a in range(cand.shape[0]):
        for j in range(cand.shape[1]):
            d = int(cand[a, j]) - first_doc
            if int(cand[a, j]) < 0 or not 0 <= d < n_docs:
                continue
            lists = list_ids[int(off[d]):int(off[d + 1])].long()
            if keep is not None:
                lists = lists[keep[a, lists]]
            if lists.numel():
                out[a, j] = s[a, lists, :lq].max(0).values.sum()
    return out


def interaction_loop(s, keep, list_ids, offsets, cand, lq: int, first_doc: int = 0) -> List[List[float]]:
    """`interaction` restated with scalar loops."""
    out = []
    for a in range(cand.shape[0]):
        row = []
        for j in range(cand.shape[1]):
            d = int(cand[a, j]) - first_doc
            if int(cand[a, j]) < 0 or not 0 <= d < len(offsets) - 1:
                row.append(-math.inf)
                continue
            best = [None] * lq
            for r in range(int(offsets[d]), int(offsets[d + 1])):
                c = int(list_ids[r])
                if keep is not None and not bool(keep[a, c]):
                    continue
                for i in range(lq):
                    v = float(s[a, c, i])
                    best[i] = v if best[i] is None else max(best[i], v)
            row.append(-math.inf if best[0] is None else sum(best))
        out.append(row)
    return out


def topk(scores: torch.Tensor, ids: torch.Tensor, k: int):
    """topk_merge: per query the k best under (score desc, id asc), void scores (NaN, -inf, <= -FLT_MAX) dropped,
    tail (-FLT_MAX, -1)."""
    out_s = torch.full((scores.shape[0], k), -FLT_MAX, dtype=torch.float64)
    out_i = torch.full((scores.shape[0], k), -1, dtype=torch.int64)
    for a in range(scores.shape[0]):
        pairs = [(float(s), int(i)) for s, i in zip(scores[a], ids[a]) if s == s and s > -FLT_MAX]
        top = sorted(pairs, key=lambda t: (-t[0], t[1]))[:k]
        for e, (s, i) in enumerate(top):
            out_s[a, e], out_i[a, e] = s, i
    return out_s, out_i


def exact_scores(q: torch.Tensor, store: torch.Tensor, offsets, cand: torch.Tensor, first_doc: int = 0) -> torch.Tensor:
    """fp64 max-sim of every candidate against the store rows (void: -inf)."""
    off = [int(v) for v in offsets]
    out = torch.full(cand.shape, -math.inf, dtype=torch.float64)
    qd = q.double()
    for a in range(cand.shape[0]):
        for j in range(cand.shape[1]):
            d = int(cand[a, j]) - first_doc
            if int(cand[a, j]) >= 0 and 0 <= d < len(off) - 1 and off[d + 1] > off[d]:
                out[a, j] = (qd[a] @ store[off[d]:off[d + 1]].double().T).max(-1).values.sum()
    return out


def search(q, cents, probes, store, offsets, list_ids, plists, ndocs: int, t_cs: float, top_n: int, first_doc: int = 0):
    """The whole pipeline on one rank: (scores, ids) [Nq, top_n].  probes [Nq, Lq * nprobe] (padding tokens -1)."""
    lq = q.shape[1]
    s, keep = centroid_scores(q, cents, t_cs)
    n_docs = len(offsets) - 1
    cap = max(1, min(n_docs, probes.shape[1] * max([len(p) for p in plists] + [0])))
    cand = candidates(probes, plists, cap, first_doc)
    _, c1 = topk(interaction(s, keep, list_ids, offsets, cand, lq, first_doc), cand, ndocs)
    _, c2 = topk(interaction(s, None, list_ids, offsets, c1, lq, first_doc), c1, ndocs // 4)
    return topk(exact_scores(q, store, offsets, c2, first_doc), c2, top_n)
