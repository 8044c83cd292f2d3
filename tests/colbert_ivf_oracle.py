"""CPU restatement of stage 1 of ColBERT retrieval with an inverted-file token index (retrieval.ColBERTIVFIndexer):
every live query token keeps its k' best rows of the union of its probed lists, as passage ids, and a query's
candidates are the de-duplicated union over its tokens.  Test infrastructure: plain torch on the CPU, no library call."""
from __future__ import annotations

from typing import Dict, List

import torch


def layout(assign: torch.Tensor, nlist: int):
    """(row_index, list_offsets) by a plain loop: list by list, the rows assigned to it in ascending order."""
    rows: List[int] = []
    off = [0]
    for l in range(nlist):
        rows += [r for r in range(len(assign)) if int(assign[r]) == l]
        off.append(len(rows))
    return torch.tensor(rows, dtype=torch.int64), torch.tensor(off, dtype=torch.int64)


def probed_rows(assign: torch.Tensor, probes_of_token) -> torch.Tensor:
    """Bool mask of the rows whose list is one of the token's probes (ids outside [0, nlist) probe nothing)."""
    p = torch.as_tensor(probes_of_token, dtype=torch.int64)
    return torch.isin(assign, p[p >= 0])


def candidates_loop(scores: torch.Tensor, live: torch.Tensor, row_pid: torch.Tensor, assign: torch.Tensor,
                    probes: torch.Tensor, kp: int, cap: int) -> List[Dict[int, float]]:
    """scores [Nq, Lq, T] token-row scores, live [Nq, Lq], row_pid [T] passage id of every row, assign [T] list id of
    every row, probes [Nq, Lq, nprobe].  Per query {passage: best single-token score}: per live token the k' best
    probed rows under (score desc, passage id asc), union, the `cap` best passages (ties by id)."""
    out = []
    for a in range(scores.shape[0]):
        best: Dict[int, float] = {}
        for t in range(scores.shape[1]):
            if not bool(live[a, t]):
                continue
            probed = set(int(x) for x in probes[a, t] if x >= 0)
            hits = [(float(scores[a, t, r]), int(row_pid[r])) for r in range(scores.shape[2]) if int(assign[r]) in probed]
            for s, p in sorted(hits, key=lambda h: (-h[0], h[1]))[:kp]:
                if p not in best or s > best[p]:
                    best[p] = s
        out.append(dict(sorted(best.items(), key=lambda kv: (-kv[1], kv[0]))[:cap]))
    return out


def candidates(scores: torch.Tensor, live: torch.Tensor, row_pid: torch.Tensor, assign: torch.Tensor,
               probes: torch.Tensor, kp: int, cap: int) -> List[Dict[int, float]]:
    """candidates_loop with tensor operations per token (fast enough for the GPU tests' sizes)."""
    out = []
    for a in range(scores.shape[0]):
        best: Dict[int, float] = {}
        for t in range(scores.shape[1]):
            if not bool(live[a, t]):
                continue
            m = probed_rows(assign, probes[a, t])
            s, pid = scores[a, t][m], row_pid[m]
            order = sorted(range(len(s)), key=lambda i: (-float(s[i]), int(pid[i])))[:kp]
            for i in order:
                p, v = int(pid[i]), float(s[i])
                if p not in best or v > best[p]:
                    best[p] = v
        out.append(dict(sorted(best.items(), key=lambda kv: (-kv[1], kv[0]))[:cap]))
    return out
