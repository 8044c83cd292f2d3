"""Shared cases of the BERT-width kernel-pooling training tests (no GPU): the shape matrix that runs every compiled
instantiation of the wide tensor-core backward, and its cases.

At 512 < D <= 1024 with D % 64 == 0 (BERT-base 768, BERT-large 1024), Lq <= 32 and K <= 32, the training forward
``kernel_pool_ts_kernel<KB, true>`` saves its cosines and norms, and the backward runs two kernels
(csrc/kernel_pool_wide.cu):

- ``kp_wide_g_kernel<KB, GATE>``: the G pass, one CTA per pair.  KB follows the tensor-core rule of
  kernel_pool_cases.tc_kb (11, 21 exact; else 12 / 24 / 32); GATE when a document gate is given.
- ``kp_wide_grad_kernel``: the two gradient GEMMs per (pair, 64-feature block); no template parameters.

The inputs, the fp64 reference and the error measure are those of kernel_pool_cases / test_kernel_pool_envelope_gpu."""
from __future__ import annotations

from dataclasses import dataclass

import torch

import kernel_pool_cases as C
from oracle import interaction_oracle as O

G_PASS, GRAD = "kp_wide_g_kernel", "kp_wide_grad_kernel"
KERNELS = (G_PASS, GRAD)


def wide_ok(Lq: int, Ld: int, D: int, K: int) -> bool:
    """kp_wide_shape_ok, csrc/kernel_pool_wide.cu."""
    return 1 <= Lq <= 32 and Ld >= 1 and 1 <= K <= 32 and 512 < D <= 1024 and D % 64 == 0


def g_inst(K: int, gate: bool) -> str:
    return C.inst(G_PASS, C.tc_kb(K), gate)


@dataclass(frozen=True)
class Row:
    B: int
    Lq: int
    Ld: int
    D: int
    K: int
    knrm: bool          # KNRM form: no alpha, log_scale 0.01, the KNRM kernel set with its sigma = 1e-4 exact-match kernel
                        # (and no exact matches: no_exact_matches)
    empty_doc: bool     # the last pair's document is fully masked
    seed: int           # chosen so that no live alpha S lies within 1 % of the 1e-10 floor
    why: str

    @property
    def shape(self):
        return self.B, self.Lq, self.Ld, self.D, self.K

    @property
    def claims(self):
        """Each row runs with and without a document gate."""
        return tuple(sorted({g_inst(self.K, False), g_inst(self.K, True), GRAD}))

    def __str__(self):
        return (f"B{self.B}-Lq{self.Lq}-Ld{self.Ld}-D{self.D}-K{self.K}" + ("-knrm" if self.knrm else "")
                + ("-emptydoc" if self.empty_doc else ""))


T, F = True, False
MATRIX = (
    Row(3, 1, 1, 576, 1, F, F, 11, "one query term, one document term, one live kernel in the 12-slot G pass"),
    Row(4, 17, 40, 768, 11, F, T, 12, "exact <11> (TK, TK-Sparse); a fully masked document"),
    Row(4, 30, 200, 768, 11, T, F, 13, "KNRM over BERT-base at the reference's token shape: sigma 1e-4 exact-match kernel"),
    Row(140, 8, 40, 768, 12, F, F, 14, "exact <12>; B > 132 pairs"),
    Row(3, 30, 200, 1024, 13, F, T, 15, "padded <24>; BERT-large; a fully masked document"),
    Row(2, 32, 2000, 768, 21, F, F, 16, "exact <21>; Lq = 32 and Ld = 2000: 32 document tiles"),
    Row(3, 32, 1000, 576, 24, F, F, 17, "exact <24>; 16 document tiles, the last one partial"),
    Row(2, 17, 1000, 1024, 25, F, F, 20, "padded <32>; BERT-large"),
    Row(3, 30, 200, 768, 32, T, F, 23, "every kernel slot live, KNRM form"),
)

CLAMP_KS = (5, 11, 21, 22, 31)
CLAMP_SHAPE = (6, 8, 60, 768)   # B, Lq, Ld, D


def no_exact_matches(d: torch.Tensor, seed: int) -> torch.Tensor:
    """Fresh document embeddings (padding rows still hold data).  At an exact match the sigma = 1e-4 kernel's gradient
    (mu - c) / sigma^2 turns a cosine rounding error of 1e-7 into 10 times its coefficient: the fp32 arithmetic of the
    reference itself cannot reproduce fp64 there (test_kernel_pool_gpu.py keeps that kernel away from near-matches too).
    Without matches every activation of that kernel underflows to 0 and its S sits at the clamp floor, as in KNRM on
    text whose query terms do not occur in the document."""
    g = torch.Generator().manual_seed(seed + 1000)
    return torch.randn(d.shape, generator=g) * 0.4


def row_case(row: Row, gate: bool) -> C.Case:
    c = C.make_case(*row.shape, seed=row.seed + (7 if gate else 0), knrm=row.knrm, gate=gate)
    if row.knrm:   # knrm.py:101-131: mu 1.0 with sigma 1e-4, then evenly spaced bins
        c.mu = torch.tensor(O.knrm_kernel_mus(row.K))
        c.sigma = torch.tensor(O.knrm_kernel_sigmas(row.K))
        c.d = no_exact_matches(c.d, row.seed)
    if row.empty_doc:
        c.dm[-1] = 0.0
    return c


def clamp_case(K: int) -> C.Case:
    """IDCM's form (kernel_pool_cases.clamp_case) at D = 768: normalised embeddings, alpha, a 1e-4 floor, the kernel at
    mu = -0.9 given the narrowest sigma so that its activations fall far below the floor."""
    c = C.make_case(*CLAMP_SHAPE, K, seed=900 + K, normalise=True)
    lo = int(torch.argmin(c.mu))
    s = int(torch.argmin(c.sigma))
    c.sigma[lo], c.sigma[s] = c.sigma[s].item(), c.sigma[lo].item()
    return c
