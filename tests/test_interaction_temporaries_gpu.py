"""Operands the backward wrappers copy into a temporary (a strided view, a half-precision gradient) give the same
gradients, bit for bit, as contiguous fp32 operands.  Several such temporaries are built for one launch; each must
still hold its data when the kernel reads it, not a later temporary's that took over its allocator block."""
import pytest
import torch

import tkl_oracle as T
from matchmaker_b200 import interaction
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _strided(x: torch.Tensor, dtype=None) -> torch.Tensor:
    """x's values (cast to dtype) in a non-contiguous view: every other element of a wider buffer."""
    wide = torch.zeros(*x.shape, 2, dtype=dtype or x.dtype, device=x.device)
    wide[..., 0] = x
    return wide[..., 0]


def _same(a, b):
    for i, (x, y) in enumerate(zip(a, b)):
        assert (x is None and y is None) or torch.equal(x, y), f"output {i} differs"


@pytest.mark.parametrize("saved", [False, True], ids=["ffma", "saved"])
def test_kernel_pool_bwd_strided_and_half_operands(saved):
    # small enough that every temporary of the call comes from the allocator's smallest block size
    B, Lq, Ld, D = 2, 3, 20, 32
    mu, sg = (torch.tensor(v, device=DEV) for v in O.tk_21_kernels())
    K = mu.numel()
    g = torch.Generator().manual_seed(31)
    w, alpha = ((torch.rand(K, generator=g) - 0.5).to(DEV), (torch.rand(K, generator=g) + 0.5).to(DEV))
    q, d, qm, dm = (t.to(DEV) for t in O.synth_kernel_pool_inputs(B, Lq, Ld, D, seed=32))
    fwd = interaction.kernel_pool(q, d, qm, dm, mu, sg, w, alpha=alpha, want_per_kernel_query=True,
                                  save_for_backward=saved)
    S, extra = fwd["per_kernel_query"], {"saved": fwd["saved"]} if saved else {}
    gout = _strided(torch.randn(B, generator=g).to(DEV), torch.float16)
    got = interaction.kernel_pool_bwd(q, d, qm, dm, mu, sg, w, alpha, _strided(S), gout, **extra)
    ref = interaction.kernel_pool_bwd(q, d, qm, dm, mu, sg, w, alpha, S.contiguous(), gout.float().contiguous(), **extra)
    _same(got, ref)


@pytest.mark.parametrize("sat", ["embedding", "log"])
def test_tkl_bwd_strided_operands(sat):
    B, Lq, D, K, C = 2, 5, 32, 11, 1
    W = (C * 40 - 30) // 2 + 1
    g = torch.Generator().manual_seed(41)
    q, chunks = torch.randn(B, Lq, D, generator=g).to(DEV), torch.randn(B * C, 40, D, generator=g).to(DEV)
    params = {k: v.to(DEV) for k, v in T.covering_params(K, D, g).items()}
    sp, red = T.sat_args(params, sat)
    top_idx = torch.tensor([[0, W - 1, W // 2]] * B, device=DEV)
    orig = (torch.rand(B, W, generator=g) + 0.5).to(DEV)
    gout = torch.randn(B, generator=g).to(DEV)

    def bwd(top_idx, orig, gout):
        return interaction.tkl_bwd(q, torch.ones(B, Lq, device=DEV), chunks, torch.ones(B * C, 40, device=DEV),
                                   torch.ones(B * C, dtype=torch.bool, device=DEV), C, params["mu"], params["sigma"],
                                   params["dense_weight"], sat, sp, red, params["chunk_scoring"], top_idx, orig, gout)

    _same(bwd(_strided(top_idx), _strided(orig), _strided(gout)), bwd(top_idx, orig, gout))
