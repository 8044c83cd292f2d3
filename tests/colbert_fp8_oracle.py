"""CPU restatement of the E4M3 token store (DESIGN 3.4i) for the tests of ``interaction.fp8_*``,
``interaction.maxsim_store`` / ``flat_ip_topk`` / ``ivf_search`` over e4m3 tensors and the fp8 ColBERT indexers.
Test infrastructure: plain Python and torch on the CPU, no library call.

- scale rule: the largest integer s with A * 2^s <= 448, found by stepping from a float estimate and checked with
  exact ldexp; 0 when A == 0; a non-finite A raises;
- stored value: torch's CPU cast to float8_e4m3fn of the fp32 value x * 2^s (taken exactly in fp64 first);
- scores: fp64 products and sums of the stored values (the scaled domain), unscaled by 2^-(s_q + s_d).  Subnormal
  stored values (m * 2^-9) count as they are: the FP8 tensor cores keep them (tests/test_maxsim_envelope_gpu.py)."""
from __future__ import annotations

import math

import torch

E4M3_MAX = 448.0


def scale_log2(amax: float) -> int:
    if not math.isfinite(amax):
        raise ValueError(f"non-finite maximum {amax}")
    if amax == 0.0:
        return 0
    s = int(math.floor(math.log2(E4M3_MAX / amax)))
    while math.ldexp(amax, s + 1) <= E4M3_MAX:
        s += 1
    while math.ldexp(amax, s) > E4M3_MAX:
        s -= 1
    return s


def quantize(x: torch.Tensor, s: int) -> torch.Tensor:
    """e4m3(x * 2^s) for one scale s."""
    return (x.double() * 2.0 ** s).float().to(torch.float8_e4m3fn)


def quantize_queries(q: torch.Tensor):
    """Per query of q [N, Lq, dim]: (e4m3 values, scales [N]) with each query's own scale."""
    s = [scale_log2(float(q[n].double().abs().max())) for n in range(q.shape[0])]
    return torch.stack([quantize(q[n], s[n]) for n in range(q.shape[0])]), torch.tensor(s, dtype=torch.int64)


def token_scores(q8: torch.Tensor, store8: torch.Tensor) -> torch.Tensor:
    """[N, Lq, T] fp64 sums of products of the stored values."""
    return torch.einsum("nld,td->nlt", q8.double(), store8.double())


def token_mass(q8: torch.Tensor, store8: torch.Tensor) -> torch.Tensor:
    """[N, Lq, T] sum_k |q_k d_k|: the scale of the accumulation error of each token product."""
    return torch.einsum("nld,td->nlt", q8.double().abs(), store8.double().abs())


def maxsim_store(q8: torch.Tensor, store8: torch.Tensor, offsets, max_doc_len: int, c: float):
    """(scores [N, n_docs] fp64 in the scaled domain, bound [N, n_docs]) of forward_aggregation over the stored values,
    reading at most max_doc_len rows per passage; -inf for passages without rows.  The bound: per query token
    c * max_j mass[j] (the max of values each off by at most c * mass[j] is off by at most the largest of them),
    plus the fp32 sum of the Lq token maxima (2^-22 of their absolute sum)."""
    ts, ms = token_scores(q8, store8), token_mass(q8, store8)
    off = [int(v) for v in offsets]
    n_docs = len(off) - 1
    out = torch.full((q8.shape[0], n_docs), -math.inf, dtype=torch.float64)
    tol = torch.zeros((q8.shape[0], n_docs), dtype=torch.float64)
    for d in range(n_docs):
        a = off[d]
        b = min(off[d + 1], a + max_doc_len)
        if b > a:
            mx = ts[:, :, a:b].max(-1).values
            out[:, d] = mx.sum(-1)
            tol[:, d] = c * ms[:, :, a:b].max(-1).values.sum(-1) + 2.0 ** -22 * mx.abs().sum(-1)
    return out, tol
