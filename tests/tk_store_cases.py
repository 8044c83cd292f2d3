"""Shared pieces of the TK store tests: a seeded ragged store, the padded gather the store mode must reproduce, and
the store scoring restated over the fp64 TK / TK-Sparse oracles."""
from __future__ import annotations

from typing import Optional

import torch

from oracle import interaction_oracle as O


def make_store(lengths, D: int, seed: int, gate_zeros: bool = False):
    """(store [sum(lengths), D] fp32, doc_offsets [n + 1] int64, gate [rows] fp32 in (0.2, 1.2], with every third row 0
    when gate_zeros)."""
    g = torch.Generator().manual_seed(seed)
    lengths = torch.tensor(lengths, dtype=torch.int64)
    off = torch.zeros(len(lengths) + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(lengths, 0)
    n = int(off[-1])
    store = torch.randn(n, D, generator=g)
    gate = torch.rand(n, generator=g) + 0.2
    if gate_zeros:
        gate[::3] = 0.0
    return store, off, gate


def gather_padded(store, off, pair_d, Ld: int, gate: Optional[torch.Tensor] = None):
    """The passages of the pairs in the padded layout: d [P, Ld, D] (zeros past a passage), d_mask [P, Ld] and the gate
    [P, Ld] (zeros past a passage); a pair with pair_d < 0 gets an empty passage."""
    P, D = len(pair_d), store.shape[1]
    d = torch.zeros(P, Ld, D, dtype=store.dtype, device=store.device)
    dm = torch.zeros(P, Ld, dtype=torch.bool, device=store.device)
    dg = torch.zeros(P, Ld, dtype=store.dtype, device=store.device)
    for p, di in enumerate(pair_d.tolist()):
        if di < 0:
            continue
        a, b = int(off[di]), int(off[di + 1])
        L = min(b - a, Ld)
        d[p, :L] = store[a:a + L]
        dm[p, :L] = True
        if gate is not None:
            dg[p, :L] = gate[a:a + L]
    return d, dm, (dg if gate is not None else None)


def store_oracle(q, q_mask, store, off, pair_q, pair_d, mu, sigma, alpha, weight, gate=None):
    """fp64 store scoring, pair by pair: the passage's rows as one unpadded document of the TK (or, with a gate,
    TK-Sparse) oracle; -inf for pair_d < 0 and empty passages."""
    out = torch.empty(len(pair_q), dtype=torch.float64)
    for p, (qi, di) in enumerate(zip(pair_q.tolist(), pair_d.tolist())):
        a, b = (int(off[di]), int(off[di + 1])) if di >= 0 else (0, 0)
        if b <= a:
            out[p] = float("-inf")
            continue
        qq, qm = q[qi:qi + 1].double(), q_mask[qi:qi + 1].double()
        dd = store[a:b].unsqueeze(0).double()
        dm = torch.ones(1, b - a, dtype=torch.float64)
        if gate is None:
            s, _ = O.kernel_pool_tk(qq, dd, qm, dm, mu.double(), sigma.double(), alpha.double(), weight.double())
        else:
            s, _ = O.kernel_pool_tk_sparse(qq, dd, qm, dm, gate[a:b].unsqueeze(0).double(), mu.double(), sigma.double(),
                                           alpha.double(), weight.double())
        out[p] = s[0]
    return out


def kernels(K: int):
    """The reference's kernel set of K kernels (knrm.py:88-111, which TK's configs use too)."""
    return torch.tensor(O.knrm_kernel_mus(K)), torch.tensor(O.knrm_kernel_sigmas(K))
