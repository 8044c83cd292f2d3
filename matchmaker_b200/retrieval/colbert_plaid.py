"""PLAID centroid-interaction search over a ColBERT IVF token index (``colbert_plaid_ndocs``, DESIGN 3.4j).

PLAID (Santhanam et al., "PLAID: An Efficient Engine for Late Interaction Retrieval", CIKM 2022) replaces the token
scan of stage 1 by scores computed from the list (centroid) ids of a passage's rows alone.  Per rank and batch of
queries q [Nq, Lq, dim], enqueued on the current stream without a host synchronisation:

1. centroid scores: S[q][c][i] = fp16_rn(fp32 sum_d fp16(q[i][d]) * fp16(centroid[c][d])) and a keep bit per
   (query, centroid), set when the max over the query's live tokens of S is >= t_cs (``interaction.plaid_centroid_scores``);
   every live token probes its nprobe lists (``IVFIndexer.coarse``), all-zero padding tokens probe nothing;
2. candidates: the union over the probed lists of the passages that own a row of the list, ascending
   (``interaction.plaid_candidates``), at a static width ``cap = min(local passages, Lq * nprobe * longest passage
   list)``, which bounds the union exactly: nothing is truncated and the shapes stay fixed;
3. pruned centroid interaction: sum over i of the max over the passage's rows whose centroid is kept of S (-inf when
   none is), then the ``ndocs`` best;
4. full centroid interaction (every row) of those, then the ``ndocs // 4`` best;
5. the store's exact max-sim of those, then the ``top_n`` best, unscaled; across ranks ``all_gather_merge``.

Every selection is ``topk_merge`` under (score desc, id asc).  Queries and centroids are cast to fp16 for S whatever
the store format: with fp32 storage only the approximate stages 1-4 see fp16.

The layout gives what the kernels read, built with torch ops whenever the indexer sets its layout (``index()``,
``load()`` then ``index()``, the residual ``load()``) and never saved:
- the passage lists: list l holds the local passages ``plist_pids[plist_offsets[l]:plist_offsets[l+1]]`` (int32,
  ascending).  ``row_index`` is ascending within a list and the store is in passage order, so the passages of the
  list's rows are non-decreasing and the list is their runs;
- the list of every store row (int32): the residual store's own ``list_ids``, else built from the layout (4 bytes per
  row, only for an indexer configured for PLAID).

Each rank keeps its own ``ndocs`` survivors, as each rank keeps its own candidate cap in the token-scan search.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch

from .. import _lib, interaction

MIN_NDOCS, MAX_NDOCS = 4, 4096
DEFAULT_THRESHOLD = 0.45      # t_cs: ColBERTv2 / PLAID's default centroid score threshold
WORKSPACE_CAP = interaction.IVF_WORKSPACE_CAP   # device scratch of one query batch


def config_keys(config) -> Optional[Tuple[int, float]]:
    """(ndocs, t_cs) of a config that enables PLAID search (``colbert_plaid_ndocs``), else None.  Raises on values
    outside the envelope: 4 <= ndocs <= 4096, t_cs not NaN (-inf keeps every centroid)."""
    ndocs = config.get("colbert_plaid_ndocs")
    t_cs = config.get("colbert_plaid_centroid_score_threshold")
    if ndocs is None:
        if t_cs is not None:
            raise _lib.MatchmakerB200Error("colbert_plaid_centroid_score_threshold needs colbert_plaid_ndocs")
        return None
    ndocs = int(ndocs)
    if not MIN_NDOCS <= ndocs <= MAX_NDOCS:
        raise _lib.MatchmakerB200Error(f"colbert_plaid_ndocs must be in [{MIN_NDOCS}, {MAX_NDOCS}], got {ndocs}")
    t_cs = DEFAULT_THRESHOLD if t_cs is None else float(t_cs)
    if math.isnan(t_cs):
        raise _lib.MatchmakerB200Error("colbert_plaid_centroid_score_threshold is NaN")
    return ndocs, t_cs


def check_envelope(nlist: int, dim: int):
    if not 1 <= nlist <= interaction.PLAID_MAX_NLIST:
        raise _lib.MatchmakerB200Error(f"PLAID search needs nlist <= 2^18, got {nlist}")
    if dim % 64 or not 64 <= dim <= 1024:
        raise _lib.MatchmakerB200Error(f"PLAID search needs token_dim % 64 == 0 and 64 <= token_dim <= 1024, got {dim}")


def list_positions(list_offsets: torch.Tensor) -> torch.Tensor:
    """The list of every list position [list_offsets[-1]] int64."""
    nlist = list_offsets.numel() - 1
    counts = list_offsets[1:] - list_offsets[:-1]
    return torch.repeat_interleave(torch.arange(nlist, device=list_offsets.device), counts)


def passage_lists(row_index: torch.Tensor, list_offsets: torch.Tensor, row_pid: torch.Tensor):
    """(plist_offsets [nlist + 1] int64, plist_pids int32, longest passage list) of a layout: list l holds the distinct
    passages (row_pid of its rows, local ids) of its rows, ascending.  Needs row_pid[row_index] non-decreasing within
    every list (ascending rows of a passage-ordered store)."""
    nlist = list_offsets.numel() - 1
    pos_list = list_positions(list_offsets)
    pid = row_pid[row_index]
    new = torch.ones_like(pid, dtype=torch.bool)
    if pid.numel() > 1:
        new[1:] = (pid[1:] != pid[:-1]) | (pos_list[1:] != pos_list[:-1])
    counts = torch.bincount(pos_list[new], minlength=nlist)
    plist_offsets = torch.zeros(nlist + 1, dtype=torch.int64, device=row_index.device)
    plist_offsets[1:] = torch.cumsum(counts, 0)
    return plist_offsets, pid[new].to(torch.int32).contiguous(), int(counts.max().item()) if nlist else 0


def row_list_ids(row_index: torch.Tensor, list_offsets: torch.Tensor, n_rows: int) -> torch.Tensor:
    """The list of every store row [n_rows] int32 from a layout that covers the rows."""
    out = torch.empty(n_rows, dtype=torch.int32, device=row_index.device)
    out[row_index] = list_positions(list_offsets).to(torch.int32)
    return out


class PLAIDSearch:
    """The PLAID search of one ``ColBERTIVFIndexer`` (or subclass): its parameters and the structures it reads."""

    def __init__(self, ndocs: int, threshold: float):
        self.ndocs, self.threshold = ndocs, threshold
        self.plist_offsets: Optional[torch.Tensor] = None   # [nlist + 1] int64
        self.plist_pids: Optional[torch.Tensor] = None      # int32 local passage ids
        self.max_plist_len = 0
        self.list_ids: Optional[torch.Tensor] = None        # [rows] int32 list of every store row
        self.centroids: Optional[torch.Tensor] = None       # [nlist, dim] fp16

    def set_layout(self, ix):
        """Build the passage lists, the row lists and the fp16 centroids from the indexer's layout."""
        check_envelope(ix.nlist, ix.token_dim)
        n_rows = ix.row_index.numel()
        row_pid = ix.row_ids - ix.d_lo
        self.plist_offsets, self.plist_pids, self.max_plist_len = passage_lists(ix.row_index, ix.list_offsets, row_pid)
        own = getattr(ix.tokens, "list_ids", None)
        self.list_ids = own if own is not None else row_list_ids(ix.row_index, ix.list_offsets, n_rows)
        self.centroids = ix.ivf.centroids.to(torch.float16).contiguous()

    def cap(self, ix, lq: int) -> int:
        """Candidate width: the rank's passages, bounded by what Lq tokens of nprobe lists can reach."""
        return max(1, min(ix.d_hi - ix.d_lo, lq * min(ix.nprobe, ix.nlist) * self.max_plist_len))

    def workspace_bytes(self, ix, nq: int, lq: int) -> int:
        """Device scratch of a batch of nq queries: S, the keep mask, the candidate bitmap and the candidate lists (ids,
        scores and the merge's copies); 0 past the per-launch query limit."""
        if nq > interaction.PLAID_MAX_QUERIES:
            return 0
        nlist, n_docs = ix.nlist, ix.d_hi - ix.d_lo
        per_query = nlist * interaction.plaid_lqp(lq) * 2 + (nlist + 31) // 32 * 4 + (n_docs + 31) // 32 * 4 + \
            self.cap(ix, lq) * 16
        return nq * per_query

    # ------------------------------------------------------------------ stages (the benchmark times them one by one)
    def centroid_scores(self, ix, q: torch.Tensor):
        """Stage 1: (S, keep, probes [Nq, Lq * nprobe]) of queries q [Nq, Lq, dim] in the store dtype."""
        nq, lq, dim = q.shape
        s, keep = interaction.plaid_centroid_scores(q, self.centroids, self.threshold)
        toks = q.reshape(nq * lq, dim)
        pad = (toks == 0).all(dim=1, keepdim=True)
        probes = ix.ivf.coarse(toks).masked_fill(pad, -1).view(nq, -1)
        return s, keep, probes

    def candidates(self, ix, probes: torch.Tensor, lq: int) -> torch.Tensor:
        """Stage 2: the candidate passages [Nq, cap] (global ids ascending, -1 tail)."""
        return interaction.plaid_candidates(probes, self.plist_offsets, self.plist_pids, ix.d_hi - ix.d_lo,
                                            self.cap(ix, lq), ix.d_lo)

    def interaction(self, ix, s, keep, cand: torch.Tensor, lq: int, k: int):
        """Stages 3 (keep given) and 4 (keep None): centroid interaction of cand, then the k best."""
        scores = interaction.plaid_interaction(s, keep, self.list_ids, ix.offsets, cand, lq, ix.d_lo)
        return interaction.topk_merge(scores, cand, k)

    def exact(self, ix, qs: torch.Tensor, cand: torch.Tensor, top_n: int):
        """Stage 5: the store's max-sim of cand [Nq, C] (void ids -1 skipped), then the top_n best (scaled domain)."""
        nq, c = cand.shape
        pair_d = torch.where(cand >= 0, cand - ix.d_lo, torch.full_like(cand, -1))
        pair_q = torch.arange(nq, device=cand.device, dtype=torch.int32).repeat_interleave(c)
        scores = ix.tokens.maxsim(qs, ix.offsets, pair_q, pair_d, ix.max_doc_len).view(nq, c)
        return interaction.topk_merge(scores, cand, top_n)

    def search(self, ix, q: torch.Tensor, top_n: int):
        """The top_n (unscaled score, global id) of queries q [Nq, Lq, dim] on this rank, in query batches whose
        scratch fits WORKSPACE_CAP."""
        nq, lq, _ = q.shape
        qs, sq = ix.tokens.queries(q)
        b = interaction.ivf_query_batch(nq, lambda n: self.workspace_bytes(ix, n, lq), WORKSPACE_CAP)
        out_s, out_i = [], []
        for b0 in range(0, nq, b):
            b1 = min(nq, b0 + b)
            s, keep, probes = self.centroid_scores(ix, q[b0:b1])
            cand = self.candidates(ix, probes, lq)
            _, cand = self.interaction(ix, s, keep, cand, lq, self.ndocs)
            _, cand = self.interaction(ix, s, None, cand, lq, self.ndocs // 4)
            bs, bi = self.exact(ix, qs[b0:b1], cand, top_n)
            out_s.append(bs)
            out_i.append(bi)
        s, i = (out_s[0], out_i[0]) if len(out_s) == 1 else (torch.cat(out_s), torch.cat(out_i))
        return ix.tokens.unscale(s, sq), i
