"""CPU restatement of ColBERT end-to-end retrieval and of the maxP de-duplication, for the tests of
``interaction.topk_unique`` / ``interaction.maxsim_store`` / ``retrieval.ColBERTEndToEndIndexer`` /
``FlatIPIndexer.search_unique``.  Test infrastructure: plain torch on the CPU, no library call."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

FLT_MAX = 3.4028234663852886e38
CANDIDATE_CAP = 4096


def is_void(s: float) -> bool:
    return s != s or s == -math.inf or s <= -FLT_MAX


def rank_pairs(pairs: List[Tuple[float, int]], k: int) -> Tuple[List[float], List[int]]:
    """(score desc, id asc) top-k of (score, id) pairs, padded with (-FLT_MAX, -1)."""
    top = sorted(pairs, key=lambda t: (-t[0], t[1]))[:k]
    s = [t[0] for t in top] + [-FLT_MAX] * (k - len(top))
    i = [t[1] for t in top] + [-1] * (k - len(top))
    return s, i


def topk_unique(scores: torch.Tensor, ids: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per query: the k best distinct ids, each at its highest score, (score desc, id asc); void candidates (NaN,
    -inf, -FLT_MAX) dropped; tail (-FLT_MAX, -1).  scores f32 [nq, L], ids i64 [nq, L]."""
    out_s, out_i = [], []
    for row_s, row_i in zip(scores.tolist(), ids.tolist()):
        best: Dict[int, float] = {}
        for s, i in zip(row_s, row_i):
            if is_void(s):
                continue
            if i not in best or s > best[i]:
                best[i] = s
        s, i = rank_pairs([(v, key) for key, v in best.items()], k)
        out_s.append(s)
        out_i.append(i)
    return torch.tensor(out_s, dtype=torch.float32), torch.tensor(out_i, dtype=torch.int64)


def maxp_loop(res_scores, ids, top_n: int) -> List[List[Tuple[int, float]]]:
    """The ``maxP->bert_dot`` aggregation of matchmaker/dense_retrieval.py:414-427, statement for statement, with
    the passage's ``seq_ids`` position in place of ``seq_ids[s_idx]``.  res_scores / ids: the [Nq, index_hit_top_n]
    result of ``indexer.search``."""
    validation_results = []
    for sample_i in range(len(ids)):
        results = []
        current_scores = res_scores[sample_i]                     # :415
        current_ids = ids[sample_i]                               # :416
        unique_ids = set()                                        # :418
        for t, s_idx in enumerate(current_ids):                   # :420
            if s_idx in unique_ids:                               # :421
                continue
            unique_ids.add(s_idx)                                 # :423
            results.append((int(s_idx), float(current_scores[t])))  # :424
            if len(results) == top_n:                             # :425
                break
        validation_results.append(results)
    return validation_results


def token_scores(q: torch.Tensor, store: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """[Nq, Lq, T] inner products of every query token with every store row, in `dtype` over the stored values."""
    return torch.einsum("qld,td->qlt", q.to(dtype), store.to(dtype))


def accumulation_tol(q: torch.Tensor, store: torch.Tensor) -> torch.Tensor:
    """[Nq, Lq, T] bound on the fp32 accumulation error of each token product (see flat_ip_check_exact in the
    interaction oracle: random-walk bound over dim/16 accumulator updates, x4 margin)."""
    dim = q.shape[-1]
    mass = torch.einsum("qld,td->qlt", q.double().abs(), store.double().abs())
    return 4.0 * (dim / 16.0) ** 0.5 * 2.0 ** -24 * mass


def maxsim_store(q: torch.Tensor, store: torch.Tensor, offsets, dtype=torch.float32) -> torch.Tensor:
    """forward_aggregation (colbert.py:100-112) of every query against every passage of a ragged store: [Nq, n_docs],
    -inf for passages without rows."""
    ts = token_scores(q, store, dtype)
    off = [int(v) for v in offsets]
    out = torch.full((q.shape[0], len(off) - 1), -math.inf, dtype=dtype)
    for d in range(len(off) - 1):
        a, b = off[d], off[d + 1]
        if b > a:
            out[:, d] = ts[:, :, a:b].max(-1).values.sum(-1)
    return out


def row_passages(offsets) -> torch.Tensor:
    off = torch.as_tensor(offsets, dtype=torch.int64)
    return torch.repeat_interleave(torch.arange(len(off) - 1), off[1:] - off[:-1])


def candidates(q: torch.Tensor, store: torch.Tensor, offsets, token_top_k: Optional[int],
               dtype=torch.float32) -> List[Dict[int, float]]:
    """Stage 1 per query: {passage id: best single-token score} of the union of the live tokens' top-k' rows
    (all rows when token_top_k is None), capped to the CANDIDATE_CAP best passages by that score (ties by id)."""
    ts = token_scores(q, store, dtype)
    pid = row_passages(offsets).tolist()
    live = (q != 0).any(-1)
    out = []
    for a in range(q.shape[0]):
        best: Dict[int, float] = {}
        for i in range(q.shape[1]):
            if not bool(live[a, i]):
                continue
            row = ts[a, i].tolist()
            order = sorted(range(len(row)), key=lambda r: (-row[r], pid[r]))
            if token_top_k is not None:
                order = order[:token_top_k]
            for r in order:
                if pid[r] not in best or row[r] > best[pid[r]]:
                    best[pid[r]] = row[r]
        cap = CANDIDATE_CAP if token_top_k is None else min(q.shape[1] * token_top_k, CANDIDATE_CAP)
        kept = sorted(best.items(), key=lambda t: (-t[1], t[0]))[:cap]
        out.append(dict(kept))
    return out


def colbert_e2e_search(q: torch.Tensor, store: torch.Tensor, offsets, top_n: int, token_top_k: Optional[int] = None,
                       dtype=torch.float32) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exhaustive (token_top_k None) or k'-limited ColBERT end-to-end search: candidates, exact max-sim, top_n under
    (score desc, id asc); (-FLT_MAX, -1) tail."""
    full = maxsim_store(q, store, offsets, dtype)
    cands = candidates(q, store, offsets, token_top_k, dtype)
    out_s, out_i = [], []
    for a, cd in enumerate(cands):
        s, i = rank_pairs([(float(full[a, d]), d) for d in cd], top_n)
        out_s.append(s)
        out_i.append(i)
    return torch.tensor(out_s, dtype=torch.float64), torch.tensor(out_i, dtype=torch.int64)
