"""Shared cases of the all-pairs (in-batch) max-sim backward tests: integer in-batch inputs built on
``maxsim_cases.make_case``, with ties between real rows, ties with the -1000 fill, fully masked documents and queries,
for either mask indexing; the gradient written out from an explicit argmax; and fp64 torch autograd of the reference
expression (colbert.py:154-162, ``oracle.maxsim_allpairs``) and of its own-masks form.

Pair p = a * n_d + b is query a against document b.  With the reference mask indexing pair (a, b) reads mask row a
(colbert.py:158); with own masks it reads mask row b."""
from __future__ import annotations

import functools
from dataclasses import dataclass

import torch

import maxsim_cases as C
from oracle import interaction_oracle as O

FILL_DOC, TIE_DOC, REALTIE_DOC, MASKED_DOC = 1, 2, 3, 4   # documents paired with a constructed purpose


@dataclass(frozen=True)
class Spec:
    dtype: torch.dtype
    n_q: int
    n_d: int
    Lq: int
    Ld: int
    dim: int
    own: bool           # True: every document masked by its own mask; False: the reference's indexing
    seed: int

    def __str__(self):
        return (f"{C.SHORT[self.dtype]}-nq{self.n_q}-nd{self.n_d}-Lq{self.Lq}-Ld{self.Ld}-d{self.dim}-"
                f"{'own' if self.own else 'ref'}")

    @property
    def special(self) -> bool:
        """Room for the fill and fill-tie documents (rows 2 and 6 live below the tail masked in every document)."""
        return self.Ld >= 10 and self.dim >= 64 and self.n_d > TIE_DOC

    @property
    def realtie(self) -> bool:
        return self.Ld >= 10 and self.n_d > REALTIE_DOC and self.Lq >= 2


def _mask_row(s: Spec, a: int, b: int) -> int:
    return b if s.own else a


@functools.lru_cache(maxsize=None)
def make_case(s: Spec) -> C.Case:
    """Integers in [-8, 3] (every sum exact in fp32).  Where the batch has room: against token 0 of query 0, document 1
    has only real rows below -1000 (the fill wins) and document 2 one real row at exactly -1000 four rows after a masked
    row (the real row wins the tie); token 1 of query 1 meets equal maximal real rows in document 3; the last query
    (n_q >= 3) has no live token and mask row 4 none at all."""
    if not s.own:
        assert s.n_q == s.n_d, "the reference mask indexing needs n_q == n_d"
    c = C.make_case(C.Row(s.dtype, s.n_q, 1, s.n_d, s.Lq, s.Ld, s.dim, "inbatch", s.seed, (), ""))
    q, d, qm, dm = c.q.clone(), c.d.clone(), c.qm.clone(), c.dm.clone()
    g = torch.Generator().manual_seed(5000 + s.seed)
    if s.Ld < 4:   # make_case masks the last three rows of every in-batch document: give short documents live rows
        dm = (torch.rand(s.n_d, s.Ld, generator=g) > 0.3).long()
        dm[0] = 1
    if s.special:
        u = torch.full((s.dim,), 3.0)
        u[0] = 1.0
        q[0, 0] = u
        qm[0, 0] = 1
        lo = -8 * int(u.sum())
        for b in (FILL_DOC, TIE_DOC):
            for j in range(s.Ld):
                d[b, j] = C.row_with_dot(u, int(torch.randint(lo, -1000, (1,), generator=g)))
        m = _mask_row(s, 0, TIE_DOC)
        dm[m, C.TIE1000_MASKED] = 0
        dm[m, C.TIE1000_REAL] = 1
        d[TIE_DOC, C.TIE1000_REAL] = C.row_with_dot(u, -1000)
    if s.realtie:
        a = 1 if s.n_q > 1 else 0
        qm[a, 1] = 1
        w = torch.where(q[a, 1] >= 0, 3.0, -3.0)
        for j in C.REALTIE_ROWS:
            if j < s.Ld - 3:
                d[REALTIE_DOC, j] = w
                dm[_mask_row(s, a, REALTIE_DOC), j] = 1
    if s.n_q >= 3:
        qm[s.n_q - 1] = 0
    if s.n_d > MASKED_DOC:
        dm[MASKED_DOC] = 0
    pair_q, pair_d = c.pair_q, c.pair_d
    return C.Case(q, d, qm, dm, pair_q, pair_d, pair_d.clone() if s.own else pair_q.clone(), c.gout)


def poisoned(c: C.Case, s: Spec):
    """q and d with NaN / +inf / -inf in every masked query token and every document row no pair reads: rows masked in
    their own document, or, with the reference indexing, rows masked in every mask row."""
    q, d = c.q.clone(), c.d.clone()
    for k, (a, i) in enumerate((~c.qm.bool()).nonzero().tolist()):
        q[a, i] = C.POISON[k % 3]
    dead = ~c.dm.bool()
    if not s.own:
        dead = dead.all(0, keepdim=True).expand_as(dead)
    for k, (b, j) in enumerate(dead.nonzero().tolist()):
        d[b, j] = C.POISON[k % 3]
    return q, d


def oracle_grads(c: C.Case, arg: torch.Tensor, n_d: int, gout: torch.Tensor = None):
    """The gradient of sum_{a,b} g[a,b] * score[a,b] with respect to q and d, written out from the argmax [n_q * n_d, Lq]:
    grad_q[a][i] += g * d[b][r], grad_d[b][r] += g * q[a][i] for every (a, b, i) with r = argmax >= 0."""
    gout = c.gout if gout is None else gout
    gq = torch.zeros(c.q.shape, dtype=torch.float64)
    gd = torch.zeros(c.d.shape, dtype=torch.float64)
    p, i = (arg >= 0).nonzero(as_tuple=True)
    r = arg[p, i]
    a, b = p // n_d, p % n_d
    g = gout.double().reshape(-1)[p].unsqueeze(-1)
    gq.index_put_((a, i), g * c.d.double()[b, r], accumulate=True)
    gd.index_put_((b, r), g * c.q.double()[a, i], accumulate=True)
    return gq, gd


def reference_autograd(q, qm, d, dm, gout, own: bool):
    """fp64 torch autograd of oracle.maxsim_allpairs (colbert.py:154-162) or, with own masks, of
    oracle.maxsim_allpairs_own_masks: (scores [n_q, n_d], grad_q, grad_d)."""
    q = q.double().detach().requires_grad_(True)
    d = d.double().detach().requires_grad_(True)
    s = (O.maxsim_allpairs_own_masks if own else O.maxsim_allpairs)(q, qm, d, dm)
    s.backward(gout.reshape(s.shape).to(s.dtype))
    return s.detach().double(), q.grad, d.grad


H, BF, F32 = C.H, C.BF, C.F32
MATRIX = (
    Spec(H, 6, 6, 32, 127, 64, False, 101),      # queries-on-M argmax with pair_dmask; Ld 127
    Spec(BF, 5, 5, 17, 129, 128, False, 102),    # bf16 queries-on-M; Ld 129
    Spec(H, 3, 7, 32, 200, 128, True, 103),      # n_q != n_d, own masks
    Spec(BF, 7, 3, 24, 1, 64, True, 104),        # Ld 1
    Spec(F32, 4, 4, 16, 129, 64, False, 105),    # f32 (SIMT)
    Spec(F32, 1, 6, 33, 127, 100, True, 106),    # n_q = 1
    Spec(H, 5, 1, 30, 200, 100, True, 107),      # n_d = 1, dim 100
    Spec(BF, 6, 6, 30, 200, 100, False, 108),
    Spec(H, 6, 6, 30, 200, 768, False, 109),     # the reference configuration's shape
    Spec(BF, 3, 5, 74, 129, 768, True, 110),     # Lq 74: the SIMT argmax's edge at dim 768
    Spec(F32, 5, 5, 74, 200, 768, False, 111),
    Spec(F32, 4, 7, 30, 127, 768, True, 112),
    Spec(H, 1, 1, 5, 1, 128, True, 113),         # one pair, one row
    Spec(BF, 3, 3, 30, 129, 128, True, 114),
    Spec(H, 40, 40, 30, 16, 64, False, 115),     # n_q * Lq = 1200: the document gradient's (a, i) in two chunks
    Spec(BF, 2, 1100, 20, 12, 64, True, 116),    # n_d = 1100: the query gradient's documents in two chunks
)
# chunk of (a, i) entries of maxsim_allpairs_bwd_d_kernel and of documents of maxsim_allpairs_bwd_q_kernel
BWD_CHUNK = 1024
