"""The training fixtures tests/golden/train_*.npz (generator: oracle/make_golden.py, ``train_*`` families) and the drop-in
ranker classes built from them.

Every fixture holds the reference class's fp32 state dict (``sd__*``), its fp32 inputs, a seeded upstream gradient per
output (``gout__*``) and, from an fp64 forward + backward of the reference class itself on exactly those values, the
outputs (``out__*``), the gradient of every parameter that received one (``gp__*``; the others are listed in
``no_grad_params``), the input-embedding gradients (``gi__*``) and the values and gradients at the interaction stage's
inputs (``ctx__*`` / ``gctx__*``).  All tensors are stored in fp32."""
import os

import numpy as np
import torch

from conftest import GOLDEN_DIR

KERNEL_POOLING = ["train_knrm", "train_conv_knrm", "train_tk_k11", "train_tk_k21", "train_tk_sparse"]
TKL = ["train_tkl_embedding", "train_tkl_log"]
WITH_PARAMETERS = KERNEL_POOLING + TKL
ALL = WITH_PARAMETERS + ["train_colbert", "train_bert_dot"]
TKL_TRIMMED = ("positional_features_q", "positional_features_d")   # stored: the leading rows only


def load(name):
    """A training fixture: numeric arrays as torch tensors, name lists as lists of str."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    return {k: (z[k].tolist() if z[k].dtype.kind == "U" else torch.from_numpy(z[k])) for k in z.files}


def state_dict(g):
    return {k[4:]: v for k, v in g.items() if k.startswith("sd__")}


def build(name, g):
    """The drop-in class of fixture ``name`` with the fixture's parameters loaded (on the CPU)."""
    from matchmaker_b200.rankers.conv_knrm import Conv_KNRM
    from matchmaker_b200.rankers.knrm import KNRM
    from matchmaker_b200.rankers.tk import ECAI20_TK
    from matchmaker_b200.rankers.tk_sparse import CIKM20_TK_Sparse
    from matchmaker_b200.rankers.tkl import TKL_sigir20
    cfg = [int(x) for x in g["cfg"]]
    sd = state_dict(g)
    if name == "train_knrm":
        m = KNRM(cfg[0])
    elif name == "train_conv_knrm":
        m = Conv_KNRM(*cfg)
    elif name.startswith("train_tk_k"):
        emb, heads, layers, ff, max_len = cfg
        m = ECAI20_TK(emb, sd["mu"].view(-1).tolist(), sd["sigma"].view(-1).tolist(), heads, layers, ff, max_len, True, True)
    elif name == "train_tk_sparse":
        emb, heads, layers, proj, ff, max_len = cfg
        m = CIKM20_TK_Sparse(emb, sd["mu"].view(-1).tolist(), sd["sigma"].view(-1).tolist(), heads, layers, proj, ff,
                             max_len, True)
    else:
        emb, heads, layers, ff = cfg
        m = TKL_sigir20(emb, sd["mu"].tolist(), sd["sigma"].tolist(), heads, layers, ff, 2000, True, True,
                        name[len("train_tkl_"):])
        # the fixture keeps the rows of the positional features that the forward reads (the query length, one
        # extended chunk); the others are the drop-in's own
        for k in TKL_TRIMMED:
            head = sd[k]
            pf = getattr(m, k).detach().clone()
            assert torch.allclose(pf[:, :head.shape[1]], head, atol=1e-6)
            pf[:, :head.shape[1]] = head
            sd[k] = pf
    m.load_state_dict(sd, strict=True)
    return m


def inputs(g, names=("q", "d", "q_mask", "d_mask")):
    return [g[k] for k in names]


def forward(name, m, q, d, qm, dm):
    """The drop-in's training forward: the outputs that carry an upstream gradient, and the TKL window selection."""
    if name == "train_tk_sparse":
        score, stop = m(q, d, qm, dm)
        return {"score": score, "document_stop_words": stop}, None
    if name in TKL:
        score, sec = m(q, d, qm, dm, output_secondary_output=True)
        return {"score": score}, sec["top_non_overlapping_idx"]
    return {"score": m(q, d, qm, dm)}, None


class PassThrough(torch.nn.Module):
    """Encoder stand-in for ColBERT / BERT_Dot: the fixtures score given vectors, as the reference classes do with
    their forward_representation replaced by "return the vectors I was given"."""

    class _Cfg:
        hidden_size = 8

    def __init__(self):
        super().__init__()
        self.config = self._Cfg()


def pass_through(tokens, sequence_type=None):
    return tokens["vecs"]
