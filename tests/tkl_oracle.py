"""fp64 reference for the TKL backward: autograd through the oracle restatement of sigir20_tkl.py:180-286
(oracle.interaction_oracle.tkl_interaction) with the top-3 window choice taken as given.

The greedy top-3 argmax is discontinuous in the window scores.  Where two windows tie within fp32 rounding, an fp32 kernel
and the fp64 oracle may pick different ones, and their gradients are then gradients of two different functions.  Gathering
the oracle's window scores at the windows the kernel picked, with the same +-1/+-2 neighbours and clamping, gives the
function whose gradient the kernel computes; with the oracle's own choice it is the oracle's score exactly
(tests/test_tkl_bwd_cpu.py)."""
import torch

from oracle import interaction_oracle as O

NEIGHBOUR_OFFSETS = (0, -1, 1, -2, 2)   # sigir20_tkl.py:274: gathered slot 3 * j + c is window top_idx[c] + offset j
SAT_EMBEDDING_KEYS = ("sat_normer_weight", "sat_normer_bias", "saturation_linear_weight", "saturation_linear_bias",
                      "saturation_linear2_weight", "saturation_linear2_bias", "saturation_linear3_weight",
                      "saturation_linear3_bias")


def gathered_windows(top_idx: torch.Tensor, W: int) -> torch.Tensor:
    """[B, 15] window ids gathered around the top-3 windows top_idx [B, 3] (sigir20_tkl.py:274-278), clamped to [0, W)."""
    top_idx = top_idx.long()
    return torch.cat([top_idx + o for o in NEIGHBOUR_OFFSETS], dim=1).clamp(0, W - 1)


def conditional_score(orig_score: torch.Tensor, chunk_scoring: torch.Tensor, top_idx: torch.Tensor) -> torch.Tensor:
    """sum_s chunk_scoring[s] * orig_score[b, gathered window s]: the TKL score with the top-3 windows fixed to top_idx.
    ``orig_score`` [B, W] has the -9900 sentinel already mapped to 0, as the oracle's sec["orig_score"] has."""
    nb = gathered_windows(top_idx.cpu(), orig_score.shape[1])
    return (torch.gather(orig_score, 1, nb) * chunk_scoring.view(1, -1)).sum(dim=1)


def covered_rows(top_idx: torch.Tensor, packed: torch.Tensor, pieces: int) -> torch.Tensor:
    """[Nc, 40] bool: the packed chunk rows that at least one of a document's gathered windows covers (window w spans the
    document positions 2w .. 2w+29; position p lies in chunk slot p // 40).  No other row can receive gradient."""
    B = top_idx.shape[0]
    C, chunk = int(pieces), O.TKL_CHUNK
    W = (C * chunk - O.TKL_WINDOW) // 2 + 1
    pos = torch.zeros(B, C * chunk, dtype=torch.bool)
    for b, wins in enumerate(gathered_windows(top_idx.cpu(), W).tolist()):
        for w in set(wins):
            pos[b, 2 * w:2 * w + O.TKL_WINDOW] = True
    return pos.view(B * C, chunk)[packed.cpu().view(-1).bool()]


def covering_params(K: int, D: int, g: torch.Generator) -> dict:
    """TKL parameters around K RBF kernels spread evenly over [-0.9, 1.0] with sigma 0.1.  Such a kernel set has cover
    (interaction.tkl_kernel_set_covers): every cosine activates some kernel in fp32 too, so the window token count of
    sigir20_tkl.py:210 is the same in fp32 and fp64.  The kernel at mu = 1.0 gets the largest dense weight, so exact
    matches raise a window's score."""
    dense = torch.randn(K, generator=g) * 0.1
    dense[-1] = 1.0
    return {"mu": torch.linspace(-0.9, 1.0, K), "sigma": torch.full((K,), 0.1),
            "dense_weight": dense, "chunk_scoring": torch.rand(15, generator=g) + 0.5,
            "sat_emb_reduce1_weight": torch.randn(D, generator=g) * 0.3,
            "sat_normer_weight": torch.rand(2, generator=g) + 0.5, "sat_normer_bias": torch.randn(2, generator=g) * 0.1,
            "saturation_linear_weight": torch.randn(2, generator=g) * 0.5, "saturation_linear_bias": torch.tensor([3.0]),
            "saturation_linear2_weight": torch.randn(2, generator=g) * 0.2, "saturation_linear2_bias": torch.tensor([2.0]),
            "saturation_linear3_weight": torch.randn(2, generator=g) * 0.5, "saturation_linear3_bias": torch.tensor([1.0]),
            "kernel_mult0": torch.rand(K, generator=g) + 0.5}


def sat_args(params: dict, saturation: str):
    """(sat_params, sat_red_weight) in the layout of interaction.tkl_window_scores / tkl_bwd."""
    if saturation == "embedding":
        return torch.cat([params[k].reshape(-1) for k in SAT_EMBEDDING_KEYS]), params["sat_emb_reduce1_weight"]
    return params["kernel_mult0"], None


def reference_grads(q, q_mask, chunks, chunk_mask, packed, pieces, params, saturation, grad_score, top_idx=None):
    """fp64 autograd of the TKL interaction stage with the top-3 windows fixed to ``top_idx`` (None: the oracle's own).

    Returns (score [B], sec, grads): sec is the oracle's secondary output; grads holds "q", "chunks", "dense_weight",
    "chunk_scoring", "sat" (laid out as sat_args) and "sat_red" (None for "log"), all fp64."""
    leaf = {k: v.double().clone().requires_grad_(True) for k, v in params.items() if k not in ("mu", "sigma")}
    p64 = dict(leaf, mu=params["mu"].double(), sigma=params["sigma"].double())
    q64 = q.double().clone().requires_grad_(True)
    c64 = chunks.double().clone().requires_grad_(True)
    _, sec = O.tkl_interaction(q64, q_mask.double(), c64, chunk_mask.double(), packed, pieces, p64, saturation)
    choice = sec["top_non_overlapping_idx"] if top_idx is None else top_idx
    score = conditional_score(sec["orig_score"], p64["chunk_scoring"], choice)
    score.backward(grad_score.double())

    def grad(t):
        return torch.zeros_like(t) if t.grad is None else t.grad

    if saturation == "embedding":
        sat = torch.cat([grad(leaf[k]).reshape(-1) for k in SAT_EMBEDDING_KEYS])
        red = grad(leaf["sat_emb_reduce1_weight"])
    else:
        sat, red = grad(leaf["kernel_mult0"]), None
    grads = {"q": grad(q64), "chunks": grad(c64), "dense_weight": grad(leaf["dense_weight"]),
             "chunk_scoring": grad(leaf["chunk_scoring"]), "sat": sat, "sat_red": red}
    return score.detach(), {k: (v.detach() if torch.is_tensor(v) else v) for k, v in sec.items()}, grads
