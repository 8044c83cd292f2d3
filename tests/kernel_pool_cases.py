"""Shared cases of the kernel-pooling envelope tests (no GPU): the shape matrix that runs every compiled instantiation of
the four cosine + RBF kernel-pooling kernels, the seeded inputs and kernel sets, and one fp64 autograd reference.

The four kernels pick a template instantiation from the kernel count K and the shape:

- tensor-core forward ``kernel_pool_ts_kernel<KB, SAVE>`` (csrc/kernel_pool_ts.cu:459-464, :408-414): K == 11 -> 11,
  K == 21 -> 21, K <= 12 -> 12, K <= 24 -> 24, else 32; SAVE for the training forward (``save_for_backward=True``).  It
  serves queries up to 128 terms (:471-472); the training forward only the training envelope.
- tensor-core backward ``kernel_pool_bwd_tc_kernel<KB, GATE>`` (csrc/kernel_pool_bwd_wg.cu:371-382): the same K rule,
  GATE when a document gate is given; training envelope only.
- FFMA forward ``kernel_pool_fwd_simt<KB, JR>`` (csrc/kernel_pool.cu:520-523): KB 12 / 24 / 32, JR = 2 when Ld > 48.
- FFMA backward ``kernel_pool_bwd_simt<KB, NC>`` (csrc/kernel_pool.cu:567-575): the same KB, NC = 2 when D > 256 (D <= 512).

The training envelope (csrc/kernel_pool.cu:489-491) is Lq <= 32, D % 4 == 0, D <= 320, K <= 32."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from oracle import interaction_oracle as O

TS_FWD, TC_BWD, SIMT_FWD, SIMT_BWD = "kernel_pool_ts_kernel", "kernel_pool_bwd_tc_kernel", "kernel_pool_fwd_simt", "kernel_pool_bwd_simt"
KERNELS = (TS_FWD, TC_BWD, SIMT_FWD, SIMT_BWD)
TS_MAX_LQ = 128       # kernel_pool_ts.cu:471-472
SIMT_BWD_MAX_D = 512  # kernel_pool.cu:547


def inst(kernel: str, a, b) -> str:
    """Canonical instantiation name, e.g. ``kernel_pool_ts_kernel<12,true>``."""
    b = str(b).lower() if isinstance(b, bool) else b
    return f"{kernel}<{a},{b}>"


def tc_kb(K: int) -> int:
    """KB of both tensor-core kernels (kernel_pool_ts.cu:459-464, kernel_pool_bwd_wg.cu:372-382)."""
    if K in (11, 21):
        return K
    return 12 if K <= 12 else 24 if K <= 24 else 32


def simt_kb(K: int) -> int:
    """KB of both FFMA kernels (kernel_pool.cu:521-523, :567-575)."""
    return 12 if K <= 12 else 24 if K <= 24 else 32


def train_ok(Lq: int, Ld: int, D: int, K: int) -> bool:
    """kp_train_tc_shape_ok, kernel_pool.cu:489-491."""
    return 1 <= Lq <= 32 and Ld >= 1 and 1 <= K <= 32 and D >= 4 and D % 4 == 0 and D <= 320


def dispatched(Lq: int, Ld: int, D: int, K: int) -> frozenset:
    """The instantiations the envelope test runs for one shape: the tensor-core forward (inference, and training where the
    envelope holds), the tensor-core backward with and without a gate, both FFMA kernels."""
    out = set()
    if Lq <= TS_MAX_LQ:
        out.add(inst(TS_FWD, tc_kb(K), False))
    if train_ok(Lq, Ld, D, K):
        out |= {inst(TS_FWD, tc_kb(K), True), inst(TC_BWD, tc_kb(K), False), inst(TC_BWD, tc_kb(K), True)}
    out.add(inst(SIMT_FWD, simt_kb(K), 2 if Ld > 48 else 1))
    if D <= SIMT_BWD_MAX_D:
        out.add(inst(SIMT_BWD, simt_kb(K), 2 if D > 256 else 1))
    return frozenset(out)


@dataclass(frozen=True)
class Row:
    B: int
    Lq: int
    Ld: int
    D: int
    K: int
    knrm: bool       # KNRM form: no alpha, log_scale 0.01
    seed: int        # chosen so that no live alpha S lies within 2 % of the 1e-10 floor (floor_margin)
    claims: Tuple[str, ...]
    why: str

    @property
    def shape(self):
        return self.B, self.Lq, self.Ld, self.D, self.K

    @property
    def train(self) -> bool:
        return train_ok(self.Lq, self.Ld, self.D, self.K)

    def __str__(self):
        return f"B{self.B}-Lq{self.Lq}-Ld{self.Ld}-D{self.D}-K{self.K}" + ("-knrm" if self.knrm else "")


def _claims(*names):
    return tuple(sorted(names))


T, F = True, False
MATRIX = (
    Row(6, 5, 20, 36, 1, F, 68, _claims(inst(TS_FWD, 12, F), inst(TS_FWD, 12, T), inst(TC_BWD, 12, F), inst(TC_BWD, 12, T),
                                        inst(SIMT_FWD, 12, 1), inst(SIMT_BWD, 12, 1)),
        "one live kernel in the 12-slot instantiations; Ld = 20 (JR = 1)"),
    Row(4, 33, 129, 260, 5, T, 431, _claims(inst(TS_FWD, 12, F), inst(SIMT_FWD, 12, 2), inst(SIMT_BWD, 12, 2)),
        "padded <12>; Lq = 33: two query blocks on the tensor-core forward, FFMA backward; D = 260: NC = 2"),
    Row(140, 8, 49, 64, 12, F, 773, _claims(inst(TS_FWD, 12, F), inst(TS_FWD, 12, T), inst(TC_BWD, 12, F), inst(TC_BWD, 12, T),
                                            inst(SIMT_FWD, 12, 2), inst(SIMT_BWD, 12, 1)),
        "exact <12>; B > 132: every CTA walks several pairs; Ld = 49: JR = 2"),
    Row(3, 32, 1000, 320, 13, F, 1368, _claims(inst(TS_FWD, 24, F), inst(TS_FWD, 24, T), inst(TC_BWD, 24, F), inst(TC_BWD, 24, T),
                                               inst(SIMT_FWD, 24, 2), inst(SIMT_BWD, 24, 2)),
        "padded <24>; D = 320 and Lq = 32: the edges of the training envelope; 16 document tiles"),
    Row(5, 1, 1, 4, 22, T, 33, _claims(inst(TS_FWD, 24, F), inst(TS_FWD, 24, T), inst(TC_BWD, 24, F), inst(TC_BWD, 24, T),
                                       inst(SIMT_FWD, 24, 1), inst(SIMT_BWD, 24, 1)),
        "padded <24>; one query term, one document term, one 16-byte row"),
    Row(4, 128, 48, 324, 24, F, 1128, _claims(inst(TS_FWD, 24, F), inst(SIMT_FWD, 24, 1), inst(SIMT_BWD, 24, 2)),
        "exact <24>; Lq = 128: four query blocks; Ld = 48: the last JR = 1 length; D = 324 outside the training envelope"),
    Row(3, 32, 129, 256, 25, F, 545, _claims(inst(TS_FWD, 32, F), inst(TS_FWD, 32, T), inst(TC_BWD, 32, F), inst(TC_BWD, 32, T),
                                             inst(SIMT_FWD, 32, 2), inst(SIMT_BWD, 32, 1)),
        "padded <32>; D = 256: the last NC = 1 width; 128 + 1 document rows"),
    Row(3, 17, 20, 320, 31, F, 391, _claims(inst(TS_FWD, 32, F), inst(TS_FWD, 32, T), inst(TC_BWD, 32, F), inst(TC_BWD, 32, T),
                                            inst(SIMT_FWD, 32, 1), inst(SIMT_BWD, 32, 2)),
        "padded <32>; the only FFMA <32,1> forward and <32,2> backward"),
    Row(150, 12, 130, 64, 11, F, 467, _claims(inst(TS_FWD, 11, F), inst(TS_FWD, 11, T), inst(TC_BWD, 11, F), inst(TC_BWD, 11, T),
                                              inst(SIMT_FWD, 12, 2), inst(SIMT_BWD, 12, 1)),
        "regression: K = 11 (KNRM, TK, Conv-KNRM, TK-Sparse)"),
    Row(4, 30, 200, 300, 21, F, 555, _claims(inst(TS_FWD, 21, F), inst(TS_FWD, 21, T), inst(TC_BWD, 21, F), inst(TC_BWD, 21, T),
                                             inst(SIMT_FWD, 24, 2), inst(SIMT_BWD, 24, 2)),
        "regression: K = 21 (TK) at the config-2 token shape"),
    Row(3, 30, 60, 128, 32, T, 253, _claims(inst(TS_FWD, 32, F), inst(TS_FWD, 32, T), inst(TC_BWD, 32, F), inst(TC_BWD, 32, T),
                                            inst(SIMT_FWD, 32, 2), inst(SIMT_BWD, 32, 1)),
        "regression: K = 32, every slot live"),
)

# kernel counts of the clamp tests: the tensor-core KB 12, 11, 21, 24, 32 and the FFMA KB 12, 24, 32
CLAMP_KS = (5, 11, 21, 22, 31)
CLAMP_SHAPE = (6, 8, 60, 64)    # B, Lq, Ld, D
IDCM_FLOOR = 1e-4               # sigir21_idcm.py:185
DEFAULT_FLOOR = 1e-10


@dataclass
class Case:
    q: torch.Tensor
    d: torch.Tensor
    qm: torch.Tensor
    dm: torch.Tensor
    mu: torch.Tensor
    sigma: torch.Tensor
    alpha: Optional[torch.Tensor]
    weight: torch.Tensor
    gate: Optional[torch.Tensor]
    gout: torch.Tensor
    log_scale: float


def kernel_set(K: int, g: torch.Generator, knrm: bool = False):
    """Distinct mu spread over [-0.9, 1.0] (1.0 first: the exact-match kernel), distinct sigma in [0.05, 0.3] in a seeded
    permuted order (so an index slip between sigma and mu / alpha / weight changes the result), distinct alpha and weight.
    No 1e-4 sigma: KNRM's exact-match conditioning is covered by test_kernel_pool_gpu.py."""
    mu = torch.linspace(1.0, -0.9, K) if K > 1 else torch.tensor([1.0])
    sigma = torch.linspace(0.3, 0.05, K)[torch.randperm(K, generator=g)]
    alpha = None if knrm else torch.rand(K, generator=g) + 0.5
    weight = (torch.rand(K, generator=g) - 0.5) * 0.5
    return mu, sigma, alpha, weight


def make_case(B, Lq, Ld, D, K, *, seed, knrm=False, gate=False, normalise=False) -> Case:
    """Random embeddings whose padding rows hold data (only the masks keep them out), random lengths (pair 0 full), one
    exact match of a live query row in every document (but where Lq = Ld = 1), and, with ``gate``, a non-negative document gate that is exactly 0
    for about a quarter of the terms (the kernels count a negative gate as 0; the reference does not)."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, Lq, D, generator=g) * 0.4
    d = torch.randn(B, Ld, D, generator=g) * 0.4
    q_len = torch.randint(1, Lq + 1, (B,), generator=g)
    d_len = torch.randint(1, Ld + 1, (B,), generator=g)
    q_len[0], d_len[0] = Lq, Ld
    qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
    dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
    for b in range(B):
        i = int(torch.randint(0, int(q_len[b]), (1,), generator=g))
        j = int(torch.randint(0, int(d_len[b]), (1,), generator=g))
        if Lq * Ld > 1:   # in a 1 x 1 pair the match would make the cosine 1 and every q / d gradient exactly 0
            d[b, j] = q[b, i]
    if normalise:   # IDCM's ESM scorer takes L2-normalised embeddings (sigir21_idcm.py:164-178)
        q, d = torch.nn.functional.normalize(q, dim=-1), torch.nn.functional.normalize(d, dim=-1)
    mu, sigma, alpha, weight = kernel_set(K, g, knrm)
    gt = None
    if gate:
        gt = torch.rand(B, Ld, generator=g) * 1.5
        gt[torch.rand(B, Ld, generator=g) < 0.25] = 0.0
    gout = torch.randn(B, generator=g)
    return Case(q, d, qm, dm, mu, sigma, alpha, weight, gt, gout, 0.01 if knrm else 1.0)


def row_case(row: Row, gate: bool) -> Case:
    return make_case(*row.shape, seed=row.seed + (7 if gate else 0), knrm=row.knrm, gate=gate)


def clamp_case(K: int) -> Case:
    """IDCM's form: normalised embeddings, alpha, a 1e-4 floor.  The kernel at mu = -0.9 gets sigma 0.05, so that its
    activations on random cosines fall far below the floor."""
    c = make_case(*CLAMP_SHAPE, K, seed=500 + K, normalise=True)
    lo = int(torch.argmin(c.mu))
    s = int(torch.argmin(c.sigma))
    c.sigma[lo], c.sigma[s] = c.sigma[s].item(), c.sigma[lo].item()
    return c


def reference(c: Case, clamp_min: float = DEFAULT_FLOOR, bias: float = 0.0, grads: bool = True) -> Dict[str, torch.Tensor]:
    """fp64 restatement of what the kernels compute, with fp64 autograd gradients:

        S_ik = sum_j dm_j gate_j exp(-(cos_ij - mu_k)^2 / (2 sigma_k^2))
        score = sum_k w_k sum_i qm_i log_scale log(max(alpha_k S_ik, clamp_min)) + bias

    It is ecai20_tk.py:105-124 (``O.kernel_pool_tk``) with an optional alpha (KNRM, log_scale 0.01: knrm.py:52-84), an
    optional gate (cikm20_tk_sparse.py:135) and a floor and bias (sigir21_idcm.py:185-186).  Returns score, per_kernel,
    S, aS (alpha S), the gradients grad_q, grad_d, grad_alpha, grad_weight, grad_gate (None where there is no such
    input), and summed_q / summed_d (see TF32_SUMMED)."""
    q64 = c.q.double().requires_grad_(grads)
    d64 = c.d.double().requires_grad_(grads)
    w64 = c.weight.double().requires_grad_(grads)
    a64 = None if c.alpha is None else c.alpha.double().requires_grad_(grads)
    g64 = None if c.gate is None else c.gate.double().requires_grad_(grads)
    mu, sg = c.mu.double().view(1, 1, 1, -1), c.sigma.double().view(1, 1, 1, -1)
    with torch.set_grad_enabled(grads):
        cos = O.cosine_matrix(q64, d64)
        if grads:
            cos.retain_grad()
        act = torch.exp(-torch.pow(cos.unsqueeze(-1) - mu, 2) / (2 * torch.pow(sg, 2)))
        w_doc = c.dm.double() if g64 is None else c.dm.double() * g64
        S = torch.sum(act * w_doc.unsqueeze(1).unsqueeze(-1), 2)
        aS = S if a64 is None else S * a64.view(1, 1, -1)
        L = torch.log(torch.clamp(aS, min=clamp_min)) * c.log_scale * c.qm.double().unsqueeze(-1)
        per_kernel = torch.sum(L, 1)
        score = per_kernel @ w64 + bias
    out = {"score": score.detach(), "per_kernel": per_kernel.detach(), "S": S.detach(), "aS": aS.detach()}
    if grads:
        score.backward(c.gout.double())
        out.update(grad_q=q64.grad, grad_d=d64.grad, grad_weight=w64.grad, grad_alpha=None if a64 is None else a64.grad,
                   grad_gate=None if g64 is None else g64.grad)
        # the magnitude the tensor-core backward's two contractions sum before the normalisation backward cancels part of
        # it: |G| |d^| / (|q| + eps) per query-gradient element, |G|^T |q^| / (|d| + eps) per document-gradient element
        G = cos.grad.abs()
        qn, dn = c.q.double().norm(dim=-1, keepdim=True) + 1e-13, c.d.double().norm(dim=-1, keepdim=True) + 1e-13
        out["summed_q"] = torch.bmm(G, (c.d.double() / dn).abs()) / qn
        out["summed_d"] = torch.bmm(G.transpose(1, 2), (c.q.double() / qn).abs()) / dn
    return out


# The tensor-core backward feeds its contractions tf32 operands: the raw embeddings truncated (at most 2^-10 relative)
# and G rounded (2^-11).  Where the normalisation backward then cancels most of what they summed -- a query row whose
# gradient is dominated by the term of its exact match, which lies along the row itself -- that rounding is no longer
# small against the result.  Each gradient element of that kernel is therefore also allowed TF32_SUMMED times the
# magnitude summed for it (summed_q / summed_d of reference()): 2^-9, above the 1.5 * 2^-10 the operand rounding can
# reach.  DESIGN.md section 2 records the measurement.
TF32_SUMMED = 2.0 ** -9


def floor_margin(aS: torch.Tensor, qm: torch.Tensor, floor: float) -> float:
    """Smallest relative distance |alpha S - floor| / floor over the live (pair, query row, kernel) entries: above about
    1e-2, fp32 and fp64 agree on which side of the clamp every entry lies."""
    live = qm.bool().unsqueeze(-1).expand_as(aS)
    return float(((aS[live] - floor).abs() / floor).min())


def below_floor_fraction(aS: torch.Tensor, qm: torch.Tensor, floor: float) -> float:
    live = qm.bool().unsqueeze(-1).expand_as(aS)
    return float((aS[live] < floor).double().mean())


def few_term_pairs(qm: torch.Tensor, limit: int = 4) -> torch.Tensor:
    """Pairs with at most ``limit`` live query terms: the tf32 operands of the tensor-core backward are held to 3e-3 there
    (test_kernel_pool_gpu.py, test_train_pair_few_query_terms_bound)."""
    return qm.sum(1) <= limit


def activation_elements(row: Row) -> int:
    """Size of the fp64 [B, Lq, Ld, K] activation tensor the reference builds for a row."""
    return row.B * row.Lq * row.Ld * row.K

