"""Generate ``tests/golden/*.npz`` by running the reference's OWN classes.

Run in the build container (``/root/reference`` mounted):

    python -m oracle.make_golden

Each fixture stores the seeded inputs, the parameters and the outputs of the
unmodified reference code (imported through ``oracle/reference_loader.py``), and
the script asserts that ``oracle/interaction_oracle.py`` reproduces them before
writing -- that is what pins the oracle.  The fixtures are small and travel to
the GPU box, where the reference itself does not exist.

The ``train_*`` families (``python -m oracle.make_golden train_tk``) hold a
training step of each reference class in fp64: parameter, input and
interaction-stage gradients, with the oracle's backward checked against them.
"""
from __future__ import annotations

import copy
import os
import sys

import numpy as np
import torch

from . import interaction_oracle as O
from . import reference_loader as R

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def _np(d):
    out = {}
    for k, v in d.items():
        if isinstance(v, torch.Tensor):
            out[k] = v.detach().cpu().numpy()
        else:
            out[k] = np.asarray(v)
    return out


def _save(name, **arrays):
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    path = os.path.join(GOLDEN_DIR, name + ".npz")
    np.savez_compressed(path, **_np(arrays))
    print(f"wrote {path} ({os.path.getsize(path) / 1024:.1f} KiB)")


def _check(a, b, what, rtol=1e-6, atol=1e-7):
    a = torch.as_tensor(a).double()
    b = torch.as_tensor(b).double()
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert torch.allclose(a, b, rtol=rtol, atol=atol), f"{what}: oracle != reference (max abs err {err}, ref {ref})"
    print(f"  oracle == reference for {what}: max abs err {err:.3e} (|ref| max {ref:.3e})")


def golden_knrm():
    torch.manual_seed(100)
    for tag, (B, Lq, Ld, D, K) in {"small": (4, 8, 24, 32, 11), "cfg1": (32, 30, 180, 300, 11)}.items():
        ref = R.load_knrm(K)
        q, d, qm, dm = O.synth_kernel_pool_inputs(B, Lq, Ld, D, seed=1235 + Lq)
        with torch.no_grad():
            score, sec = ref.forward(q, d, qm, dm, output_secondary_output=True)
            score_plain = ref.forward(q, d, qm, dm)
        mu = ref.mu.view(-1)
        sigma = ref.sigma.view(-1)
        w = ref.dense.weight.detach().view(-1)
        o_score, o_sec = O.kernel_pool_knrm(q, d, qm, dm, mu, sigma, w)
        _check(o_score, score, f"knrm[{tag}] score")
        _check(o_score, score_plain, f"knrm[{tag}] score (no secondary)")
        _check(o_sec["per_kernel"], sec["per_kernel"], f"knrm[{tag}] per_kernel")
        _check(o_sec["cosine_matrix_masked"], sec["cosine_matrix_masked"], f"knrm[{tag}] cosine")
        assert mu.tolist() == torch.tensor(O.knrm_kernel_mus(K)).tolist()
        assert sigma.tolist() == torch.tensor(O.knrm_kernel_sigmas(K)).tolist()
        _save(f"knrm_{tag}", q=q, d=d, q_mask=qm, d_mask=dm, mu=mu, sigma=sigma, weight=w,
              score=score, per_kernel=sec["per_kernel"], query_mean_vector=sec["query_mean_vector"],
              cosine_matrix_masked=sec["cosine_matrix_masked"])


def golden_tk():
    torch.manual_seed(101)
    emb, heads, layers, ff, max_len = 40, 4, 2, 32, 64
    for tag, (mu, sigma) in {"k11": ([1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9], [0.1] * 11),
                             "k21": O.tk_21_kernels()}.items():
        ref = R.load_tk(emb, mu, sigma, heads, layers, ff, max_len, True, True)
        ref.eval()
        with torch.no_grad():
            ref.kernel_alpha_scaler.copy_(torch.rand_like(ref.kernel_alpha_scaler) + 0.5)
        B, Lq, Ld = 5, 12, 48
        q, d, qm, dm = O.synth_kernel_pool_inputs(B, Lq, Ld, emb, seed=2000 + len(mu))
        with torch.no_grad():
            score, sec = ref.forward(q, d, qm, dm, output_secondary_output=True)
            q_ctx = ref.forward_representation(q, qm, ref.positional_features_q[:, :Lq, :])
            d_ctx = ref.forward_representation(d, dm, ref.positional_features_d[:, :Ld, :])
        w = ref.kernel_bin_weights.weight.detach().view(-1)
        alpha = ref.kernel_alpha_scaler.detach().view(-1)
        o_score, o_sec = O.kernel_pool_tk(q_ctx, d_ctx, qm, dm, ref.mu.view(-1), ref.sigma.view(-1), alpha, w)
        _check(o_score, score, f"tk[{tag}] score", rtol=1e-5, atol=1e-6)
        _check(o_sec["per_kernel"], sec["per_kernel"], f"tk[{tag}] per_kernel", rtol=1e-5, atol=1e-5)
        _check(o_sec["cosine_matrix"], sec["cosine_matrix"], f"tk[{tag}] cosine")
        state = {"sd__" + k: v for k, v in ref.state_dict().items()}
        _save(f"tk_{tag}", q=q, d=d, q_mask=qm, d_mask=dm, q_ctx=q_ctx, d_ctx=d_ctx,
              mu=ref.mu.view(-1), sigma=ref.sigma.view(-1), alpha=alpha, weight=w,
              score=score, per_kernel=sec["per_kernel"], query_mean_vector=sec["query_mean_vector"],
              cosine_matrix=sec["cosine_matrix"],
              cfg=np.array([emb, heads, layers, ff, max_len]), **state)


def golden_tkl():
    torch.manual_seed(102)
    emb, heads, layers, ff = 40, 4, 1, 32
    mu = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]
    sigma = [0.1] * 11
    for sat in ("embedding", "log"):
        ref = R.load_tkl(emb, mu, sigma, heads, layers, ff, 2000, True, True, sat)
        ref.eval()
        with torch.no_grad():  # make the learned pieces non-trivial but well-conditioned
            ref.chunk_scoring.copy_(torch.rand_like(ref.chunk_scoring) + 0.5)
            ref.kernel_mult.copy_(torch.rand_like(ref.kernel_mult) + 0.5)
            ref.sat_emb_reduce1.weight.copy_(torch.randn_like(ref.sat_emb_reduce1.weight) * 0.3)
            ref.dense.weight.copy_(torch.randn_like(ref.dense.weight) * 0.1)
        B, Lq, Ld = 4, 10, 330
        g = torch.Generator().manual_seed(77)
        q = torch.randn(B, Lq, emb, generator=g) * 0.4
        d = torch.randn(B, Ld, emb, generator=g) * 0.4
        q_len = torch.tensor([10, 7, 3, 10])
        d_len = torch.tensor([330, 200, 47, 121])
        for b in range(B):  # exact matches
            d[b, 5] = q[b, 1]
            d[b, int(d_len[b]) - 3] = q[b, 0]
        qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
        dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
        q = q * qm.unsqueeze(-1)
        d = d * dm.unsqueeze(-1)
        with torch.no_grad():
            if sat == "embedding":
                score, sec = ref.forward(q, d, qm, dm, output_secondary_output=True)
            else:
                # the reference's secondary-output branch reads `sat_influencer`, which only the
                # "embedding" branch defines (sigir20_tkl.py:290) -> only the score is available
                score, sec = ref.forward(q, d, qm, dm), None
            # the pre-part of forward (sigir20_tkl.py:136-175), re-run to expose the
            # tensors that enter the interaction stage
            q_ctx, _ = ref.forward_representation(q, qm, ref.positional_features_q[:, :Lq, :])
            cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
            docs_packed = cd2[packed]
            pad_packed = cp2[packed]
            dp, _ = ref.forward_representation(docs_packed, pad_packed,
                                               ref.positional_features_d[:, :docs_packed.shape[1], :])
            doc_chunks_ctx = dp[:, O.TKL_OVERLAP:-O.TKL_OVERLAP, :].contiguous()
            doc_chunk_mask = pad_packed[:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
        if sec is not None:
            assert sec["total_chunks"] == cd2.shape[0] and sec["packed_chunks"] == docs_packed.shape[0]
        params = {
            "mu": ref.mu.detach(), "sigma": ref.sigma.detach(), "dense_weight": ref.dense.weight.detach().view(-1),
            "chunk_scoring": ref.chunk_scoring.detach().view(-1),
            "sat_emb_reduce1_weight": ref.sat_emb_reduce1.weight.detach().view(-1),
            "sat_normer_weight": ref.sat_normer.weight.detach(), "sat_normer_bias": ref.sat_normer.bias.detach(),
            "saturation_linear_weight": ref.saturation_linear.weight.detach().view(-1),
            "saturation_linear_bias": ref.saturation_linear.bias.detach(),
            "saturation_linear2_weight": ref.saturation_linear2.weight.detach().view(-1),
            "saturation_linear2_bias": ref.saturation_linear2.bias.detach(),
            "saturation_linear3_weight": ref.saturation_linear3.weight.detach().view(-1),
            "saturation_linear3_bias": ref.saturation_linear3.bias.detach(),
            "kernel_mult0": ref.kernel_mult.detach()[0].view(-1),
        }
        o_score, o_sec = O.tkl_interaction(q_ctx, qm, doc_chunks_ctx, doc_chunk_mask, packed, pieces, params, sat)
        _check(o_score, score, f"tkl[{sat}] score", rtol=1e-5, atol=1e-5)
        if sec is None:  # intermediates come from the (score-pinned) oracle for this branch
            sec = {k: o_sec[k] for k in ("orig_score", "top_non_overlapping_idx", "top_k_non_overlapping")}
        _check(o_sec["orig_score"], sec["orig_score"], f"tkl[{sat}] orig_score", rtol=1e-5, atol=1e-5)
        assert torch.equal(o_sec["top_non_overlapping_idx"], sec["top_non_overlapping_idx"])
        _check(o_sec["top_k_non_overlapping"], sec["top_k_non_overlapping"], f"tkl[{sat}] top15", rtol=1e-5, atol=1e-5)
        state = {"sd__" + k: v for k, v in ref.state_dict().items()
                 if not k.startswith("positional_features")}
        _save(f"tkl_{sat}", q=q, d=d, q_mask=qm, d_mask=dm, q_ctx=q_ctx, doc_chunks_ctx=doc_chunks_ctx,
              doc_chunk_mask=doc_chunk_mask, packed_indices=packed, chunk_pieces=np.array(pieces),
              score=score, orig_score=sec["orig_score"], top_non_overlapping_idx=sec["top_non_overlapping_idx"],
              top_k_non_overlapping=sec["top_k_non_overlapping"],
              cfg=np.array([emb, heads, layers, ff]),
              **{"p__" + k: v for k, v in params.items()}, **state)


def golden_colbert():
    cls, inst = R.load_colbert()
    # (a) fp32, masked pair scoring + unmasked aggregation + all-pairs, small
    q, d, qm, dm = O.synth_colbert_inputs(6, 1, 8, 20, 32, seed=1237, dtype=torch.float32, full_q=False)
    with torch.no_grad():
        score = inst.forward({"vecs": q.clone(), "attention_mask": qm}, {"vecs": d.clone(), "attention_mask": dm},
                             use_fp16=False)
        agg = cls.forward_aggregation(inst, q.clone(), d.clone())
        allp = cls.forward_inbatch_aggregation(inst, q.clone(), qm, d.clone(), dm)
    _check(O.maxsim_pairs(q.clone(), d.clone(), qm, dm), score, "colbert forward (masked)")
    _check(O.maxsim_pairs(q.clone(), d.clone(), None, None), agg, "colbert forward_aggregation")
    _check(O.maxsim_allpairs(q.clone(), qm, d.clone(), dm), allp, "colbert forward_inbatch_aggregation")
    _save("colbert_small", q=q, d=d, q_mask=qm, d_mask=dm, score=score, agg=agg, allpairs=allp)
    # (b) BASELINE config-3 token shape, fp16 storage upcast to fp32 like
    # dense_retrieval.py:406 (.float()), 2 queries x 3 docs
    q, d, qm, dm = O.synth_colbert_inputs(2, 3, 32, 180, 128, seed=1237, dtype=torch.float16)
    qe = q.float().repeat_interleave(3, dim=0)
    qme = qm.repeat_interleave(3, dim=0)
    with torch.no_grad():
        score = inst.forward({"vecs": qe.clone(), "attention_mask": qme},
                             {"vecs": d.float(), "attention_mask": dm}, use_fp16=False)
    _check(O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, 3), score, "colbert cfg3-shape")
    _save("colbert_cfg3", q=q, d=d, q_mask=qm, d_mask=dm, docs_per_query=np.array(3), score=score)


def golden_bert_dot():
    cls, inst = R.load_bert_dot()
    inst.eval()
    g = torch.Generator().manual_seed(1238)
    qv = torch.randn(8, 64, generator=g)
    dv = torch.randn(8, 64, generator=g)
    with torch.no_grad():
        score = inst.forward({"vecs": qv}, {"vecs": dv}, use_fp16=False)
    _check(O.dot_pairs(qv, dv), score, "bert_dot forward")
    _save("bert_dot_small", qv=qv, dv=dv, score=score)


def golden_tk_sparse():
    """CIKM20_TK_Sparse (models/published/cikm20_tk_sparse.py): full forward of the reference class; the fixture keeps the
    tensors that enter the interaction stage (contextualised embeddings + the learned document-term gate)."""
    torch.manual_seed(103)
    emb, heads, layers, proj, ff, max_len = 40, 4, 1, 16, 32, 64
    mu = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]
    sigma = [0.1] * 11
    ref = R.load_tk_sparse(emb, mu, sigma, heads, layers, proj, ff, max_len, True)
    ref.eval()
    with torch.no_grad():
        ref.kernel_alpha_scaler.copy_(torch.rand_like(ref.kernel_alpha_scaler) + 0.5)
        ref.stop_word_reducer2.bias.fill_(0.3)     # so that relu() closes the gate for a share of the document terms
    B, Lq, Ld = 6, 12, 48
    q, d, qm, dm = O.synth_kernel_pool_inputs(B, Lq, Ld, emb, seed=2100)
    with torch.no_grad():
        score, sec, stop = ref.forward(q, d, qm, dm, output_secondary_output=True)
        score_plain, stop_plain = ref.forward(q, d, qm, dm)
        q_ctx, _ = ref.forward_representation(q, qm, ref.positional_features_q[:, :Lq, :])
        d_ctx, _ = ref.forward_representation(d, dm, ref.positional_features_d[:, :Ld, :])
    assert torch.equal(score, score_plain) and torch.equal(stop, stop_plain)
    gate = stop.squeeze(1)
    assert 0.05 < float((gate[dm.bool()] == 0).float().mean()) < 0.95, "the fixture should contain closed and open gates"
    w = ref.kernel_bin_weights.weight.detach().view(-1)
    alpha = ref.kernel_alpha_scaler.detach().view(-1)
    o_score, o_sec = O.kernel_pool_tk_sparse(q_ctx, d_ctx, qm, dm, gate, ref.mu.view(-1), ref.sigma.view(-1), alpha, w)
    _check(o_score, score, "tk_sparse score", rtol=1e-5, atol=1e-6)
    _check(o_sec["per_kernel"], sec["per_kernel"], "tk_sparse per_kernel", rtol=1e-5, atol=1e-5)
    state = {"sd__" + k: v for k, v in ref.state_dict().items()}
    _save("tk_sparse", q=q, d=d, q_mask=qm, d_mask=dm, q_ctx=q_ctx, d_ctx=d_ctx, doc_gate=gate, mu=ref.mu.view(-1),
          sigma=ref.sigma.view(-1), alpha=alpha, weight=w, score=score, per_kernel=sec["per_kernel"],
          document_stop_words=stop, cfg=np.array([emb, heads, layers, proj, ff, max_len]), **state)


def golden_conv_knrm():
    """Conv_KNRM (models/conv_knrm.py): full forward of the reference class + the n-gram tensors between the
    convolutions and the 3 x 3 cross-match."""
    torch.manual_seed(104)
    emb, n_grams, K, conv_out = 24, 3, 11, 32
    ref = R.load_conv_knrm(emb, n_grams, K, conv_out)
    ref.eval()
    B, Lq, Ld = 5, 9, 40
    q, d, qm, dm = O.synth_kernel_pool_inputs(B, Lq, Ld, emb, seed=2200)
    with torch.no_grad():
        score = ref.forward(q, d, qm, dm)
        qg = [c(q.transpose(1, 2)).transpose(1, 2) for c in ref.convolutions]
        dg = [c(d.transpose(1, 2)).transpose(1, 2) for c in ref.convolutions]
    o_score, o_all = O.conv_knrm_cross_match(qg, dg, qm, dm, ref.mu.view(-1), ref.sigma.view(-1), ref.dense.weight.view(-1))
    _check(o_score, score, "conv_knrm score")
    state = {"sd__" + k: v for k, v in ref.state_dict().items()}
    _save("conv_knrm", q=q, d=d, q_mask=qm, d_mask=dm, mu=ref.mu.view(-1), sigma=ref.sigma.view(-1),
          dense_weight=ref.dense.weight.detach().view(-1), score=score, all_grams=o_all,
          cfg=np.array([emb, n_grams, K, conv_out]),
          **{f"qg{i}": t for i, t in enumerate(qg)}, **{f"dg{i}": t for i, t in enumerate(dg)}, **state)


# ----------------------------------------------------------------------------------------------------------------------
# training fixtures: forward + backward of the reference classes themselves, in fp64
#
# Each ``train_*`` fixture holds the fp32 state dict (``sd__*``), the fp32 inputs, a seeded upstream gradient per output
# (``gout__*``), and from an fp64 run of the same class on those exact values: the outputs (``out__*``), the gradient
# of every named parameter that received one (``gp__*``, the others listed in ``no_grad_params``), the input-embedding
# gradients (``gi__*``) and the values and gradients at the interaction stage's inputs (``ctx__*`` / ``gctx__*``).
# Before writing, fp64 autograd of the oracle function on ``ctx__*`` must reproduce ``gctx__*`` and the interaction
# parameters' gradients: that pins the oracle's backward to the reference's.
# ----------------------------------------------------------------------------------------------------------------------

GRAD_BAR = 2e-3                 # the GPU tests hold every gradient to 2e-3 * the tensor's largest reference entry
FP32_SHARE = GRAD_BAR / 4       # the reference's own fp32 run may use at most a quarter of that
PIN_TOL = 1e-10                 # oracle backward vs the reference's backward, both fp64 (relative to the largest entry)
FLOOR = 1e-10                   # the clamp floor of every kernel-pooling ranker's log
# Parameter-gradient entries this small relative to their tensor's largest entry are stored as exact zeros.  They are
# mathematically zero -- e.g. the key part of a transformer's in_proj_bias, since a key bias shifts every score of a
# softmax row alike -- and what the fp64 run leaves there (~1e-16 of the largest entry) is round-off whose bits depend on
# the CPU's arithmetic path, so the fixtures would not regenerate bit for bit on another machine.
ROUNDOFF = 1e-12


def _rel_err(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    scale = b.abs().max().item()
    return (a - b).abs().max().item() / scale if scale > 0 else (a - b).abs().max().item()


def _pin(got, ref, what):
    err = _rel_err(got, ref)
    assert err <= PIN_TOL, f"{what}: oracle backward != reference backward (rel err {err:.3e})"
    print(f"  oracle backward == reference for {what}: rel err {err:.1e}")


class _Retain:
    """Collects non-leaf tensors and keeps their gradients (``retain_grad``) so the backward at a stage can be read."""

    def __init__(self):
        self.t = {}

    def __call__(self, name, x):
        x.retain_grad()
        self.t[name] = x
        return x


def _train_run(ref, dtype, inputs, leaves, forward, gouts):
    """``ref`` cast to ``dtype`` in train() mode; ``inputs`` cast likewise (``leaves`` become leaf tensors that require
    grad); ``forward(model, x, retain)`` returns the outputs by name.  Backpropagates sum(out * gout) and returns
    outputs, parameter gradients (None where the reference leaves none), leaf gradients and the retained tensors."""
    m = copy.deepcopy(ref).to(dtype).train()
    for k, v in vars(m).items():   # KNRM / Conv-KNRM keep mu and sigma as plain tensor attributes, which .to() skips
        if isinstance(v, torch.Tensor) and v.is_floating_point():
            setattr(m, k, v.to(dtype))
    for p in m.parameters():
        p.grad = None
    x = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in inputs.items()}
    for k in leaves:
        x[k] = x[k].clone().requires_grad_(True)
    retain = _Retain()
    outs = forward(m, x, retain)
    total = sum((outs[k] * gouts[k].to(dtype)).sum() for k in outs)
    total.backward()
    return {"out": {k: v.detach() for k, v in outs.items()},
            "gp": {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in m.named_parameters()},
            "gi": {k: x[k].grad.detach().clone() for k in leaves},
            "ctx": {k: v.detach() for k, v in retain.t.items()},
            "gctx": {k: v.grad.detach().clone() for k, v in retain.t.items()}}


def _train_check_and_save(name, ref, inputs, leaves, forward, gouts, pin, condition, extra=None, trim=None, post=None):
    """Runs ``ref`` in fp64 and fp32, checks the fp64 run against the oracle (``pin``) and its conditioning
    (``condition``), that the fp32 run stays within FP32_SHARE of it on every tensor, and that everything is finite;
    then writes tests/golden/<name>.npz with ``extra`` (a dict, or a function of the fp64 run).  ``trim`` maps a parameter name to the leading rows that are stored of its
    value and gradient (the rest of the gradient must be exactly zero); ``post`` rewrites each run's result first."""
    trim = trim or {}
    r64 = _train_run(ref, torch.float64, inputs, leaves, forward, gouts)
    r32 = _train_run(ref, torch.float32, inputs, leaves, forward, gouts)
    if post is not None:
        post(r64)
        post(r32)
    print(f"{name}:")
    pin(r64)
    condition(r64)
    worst = {}
    for part in ("out", "gp", "gi", "ctx", "gctx"):
        for k, v in r64[part].items():
            if v is None:
                assert r32[part][k] is None, f"{name} {part}[{k}]: fp32 and fp64 disagree on whether it has a gradient"
                continue
            assert torch.isfinite(v).all(), f"{name} {part}[{k}] is not finite"
            worst[f"{part}[{k}]"] = _rel_err(r32[part][k], v)
    k_worst = max(worst, key=worst.get)
    assert worst[k_worst] <= FP32_SHARE, f"{name}: the fp32 reference run is {worst[k_worst]:.2e} off at {k_worst}"
    print(f"  fp32 reference vs fp64: worst {worst[k_worst]:.2e} at {k_worst}")
    arrays = {}
    for k, v in ref.state_dict().items():
        arrays["sd__" + k] = v[:, :trim[k]] if k in trim else v
    for k, v in r64["gp"].items():
        if v is None:
            continue
        if k in trim:
            assert (v[:, trim[k]:] == 0).all(), f"{name}: gradient of {k} beyond row {trim[k]}"
            v = v[:, :trim[k]]
        arrays["gp__" + k] = torch.where(v.abs() <= ROUNDOFF * v.abs().max(), torch.zeros_like(v), v)
    names = [n for n, _ in ref.named_parameters()]
    arrays["param_names"] = np.array(names)
    arrays["no_grad_params"] = np.array([n for n in names if r64["gp"][n] is None], dtype=f"<U{max(map(len, names))}")
    arrays.update({k: v for k, v in inputs.items()})
    arrays.update({"gout__" + k: v for k, v in gouts.items()})
    for part in ("out", "gi", "ctx", "gctx"):
        arrays.update({f"{part}__{k}": v for k, v in r64[part].items()})
    arrays.update((extra(r64) if callable(extra) else extra) or {})
    # stored in fp32: their rounding (6e-8 relative) is far below the GPU tests' bars, and it halves the files
    arrays = {k: (v.float() if isinstance(v, torch.Tensor) and v.dtype == torch.float64 else v) for k, v in arrays.items()}
    _save(name, **arrays)


def _seeded(seed, *shapes):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g) for s in shapes]


def _leaf64(t):
    return t.detach().double().clone().requires_grad_(True)


def _floor_margin(per_kernel_query, q_mask, alpha=None):
    """Smallest |alpha S - floor| / floor over the live (pair, query term, kernel) entries: above 1e-2, fp32 and fp64
    agree on which side of the clamp every entry lies."""
    aS = per_kernel_query if alpha is None else per_kernel_query * alpha.view(1, 1, -1)
    live = q_mask.bool().unsqueeze(-1).expand_as(aS)
    return float(((aS[live] - FLOOR).abs() / FLOOR).min())


def _max_live_cosine(q, d, q_mask, d_mask):
    cos = O.cosine_matrix(q.double(), d.double())
    live = (q_mask.unsqueeze(-1) * d_mask.unsqueeze(1)).bool()
    return float(cos[live].max())


def _knrm_inputs(B, Lq, Ld, D, seed):
    """synth_kernel_pool_inputs with fresh document rows: no exact or near-exact matches, so the sigma = 1e-4 kernel's
    activations all underflow (at a match its gradient (mu - c) / sigma^2 turns a cosine rounding error of 1e-7 into
    10 times its coefficient, beyond what the reference's own fp32 arithmetic reproduces).  The first pair gets a
    one-term query."""
    q, d, qm, dm = O.synth_kernel_pool_inputs(B, Lq, Ld, D, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    d = torch.randn(d.shape, generator=g) * 0.4 * dm.unsqueeze(-1)
    qm[0, 1:] = 0
    q = q * qm.unsqueeze(-1)
    return q, d, qm, dm


def train_knrm():
    torch.manual_seed(110)
    K = 11
    ref = R.load_knrm(K)
    q, d, qm, dm = _knrm_inputs(4, 8, 24, 32, seed=3100)
    (gs,) = _seeded(3101, (q.shape[0],))
    inputs = {"q": q, "d": d, "q_mask": qm, "d_mask": dm}

    def forward(m, x, retain):
        return {"score": m.forward(x["q"], x["d"], x["q_mask"], x["d_mask"])}

    def pin(r):
        q64, d64, w64 = _leaf64(q), _leaf64(d), _leaf64(ref.dense.weight.view(-1))
        s, sec = O.kernel_pool_knrm(q64, d64, qm.double(), dm.double(), ref.mu.view(-1).double(),
                                    ref.sigma.view(-1).double(), w64)
        s.backward(gs.double())
        _pin(s.detach(), r["out"]["score"], "knrm score")
        _pin(q64.grad, r["gi"]["q"], "knrm grad q")
        _pin(d64.grad, r["gi"]["d"], "knrm grad d")
        _pin(w64.grad, r["gp"]["dense.weight"].view(-1), "knrm grad dense.weight")
        assert _floor_margin(sec["per_kernel_query"].detach(), qm) > 1e-2

    def condition(r):
        assert _max_live_cosine(q, d, qm, dm) < 0.99, "near-exact match for the sigma = 1e-4 kernel"

    _train_check_and_save("train_knrm", ref, inputs, ("q", "d"), forward, {"score": gs}, pin, condition,
                          extra={"cfg": np.array([K])})


def train_conv_knrm():
    torch.manual_seed(111)
    emb, n_grams, K, conv_out = 24, 3, 11, 32
    ref = R.load_conv_knrm(emb, n_grams, K, conv_out)
    q, d, qm, dm = _knrm_inputs(5, 9, 40, emb, seed=3200)
    (gs,) = _seeded(3201, (q.shape[0],))
    inputs = {"q": q, "d": d, "q_mask": qm, "d_mask": dm}

    def forward(m, x, retain):
        # conv_knrm.py:114-119 runs each convolution on the query, then on the document: keep both outputs
        calls = []
        hooks = [c.register_forward_hook(lambda mod, i, o, n=n: calls.append((n, o))) for n, c in enumerate(m.convolutions)]
        score = m.forward(x["q"], x["d"], x["q_mask"], x["d_mask"])
        for h in hooks:
            h.remove()
        assert [n for n, _ in calls] == [n for n in range(n_grams) for _ in (0, 1)]
        for j, (n, o) in enumerate(calls):
            retain(f"{'qd'[j % 2]}g{n}", o)
        return {"score": score}

    def pin(r):
        qg = [_leaf64(r["ctx"][f"qg{i}"].transpose(1, 2)) for i in range(n_grams)]
        dg = [_leaf64(r["ctx"][f"dg{i}"].transpose(1, 2)) for i in range(n_grams)]
        w64 = _leaf64(ref.dense.weight.view(-1))
        s, _ = O.conv_knrm_cross_match(qg, dg, qm.double(), dm.double(), ref.mu.view(-1).double(),
                                       ref.sigma.view(-1).double(), w64)
        s.backward(gs.double())
        _pin(s.detach(), r["out"]["score"], "conv_knrm score")
        for i in range(n_grams):
            _pin(qg[i].grad, r["gctx"][f"qg{i}"].transpose(1, 2), f"conv_knrm grad qg{i}")
            _pin(dg[i].grad, r["gctx"][f"dg{i}"].transpose(1, 2), f"conv_knrm grad dg{i}")
        _pin(w64.grad, r["gp"]["dense.weight"].view(-1), "conv_knrm grad dense.weight")
        for i in range(n_grams):
            for t in range(n_grams):
                _, sec = O.kernel_pool_knrm(qg[i].detach(), dg[t].detach(), qm.double(), dm.double(),
                                            ref.mu.view(-1).double(), ref.sigma.view(-1).double(), w64.detach()[:K])
                assert _floor_margin(sec["per_kernel_query"], qm) > 1e-2

    def condition(r):
        for i in range(n_grams):
            for t in range(n_grams):
                c = _max_live_cosine(r["ctx"][f"qg{i}"].transpose(1, 2), r["ctx"][f"dg{t}"].transpose(1, 2), qm, dm)
                assert c < 0.99, f"near-exact match between query {i + 1}-grams and document {t + 1}-grams ({c})"

    _train_check_and_save("train_conv_knrm", ref, inputs, ("q", "d"), forward, {"score": gs}, pin, condition,
                          extra={"cfg": np.array([emb, n_grams, K, conv_out])})


def _wrap_representation(m, retain, names):
    """Instance-level wrapper of ``forward_representation`` that retains the gradient of the tensor it returns (the
    first one, when it returns a pair), naming the calls in order."""
    cls_fn = type(m).forward_representation
    it = iter(names)

    def wrapped(*a, **kw):
        out = cls_fn(m, *a, **kw)
        if isinstance(out, tuple):
            return (retain(next(it), out[0]),) + tuple(out[1:])
        return retain(next(it), out)

    m.forward_representation = wrapped


def _tk_inputs(B, Lq, Ld, D, seed):
    q, d, qm, dm = O.synth_kernel_pool_inputs(B, Lq, Ld, D, seed=seed)
    qm[0, 1:] = 0   # a one-term query
    return q * qm.unsqueeze(-1), d, qm, dm


def train_tk():
    emb, heads, layers, ff, max_len = 40, 4, 2, 32, 64
    for tag, (mu, sigma) in {"k11": ([1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9], [0.1] * 11),
                             "k21": O.tk_21_kernels()}.items():
        torch.manual_seed(112 + len(mu))
        ref = R.load_tk(emb, mu, sigma, heads, layers, ff, max_len, True, True)
        with torch.no_grad():
            ref.kernel_alpha_scaler.copy_(torch.rand_like(ref.kernel_alpha_scaler) + 0.5)
            ref.mixer.fill_(0.3)
        q, d, qm, dm = _tk_inputs(5, 12, 48, emb, seed=3300 + len(mu))
        (gs,) = _seeded(3301 + len(mu), (q.shape[0],))
        inputs = {"q": q, "d": d, "q_mask": qm, "d_mask": dm}

        def forward(m, x, retain):
            _wrap_representation(m, retain, ("q_ctx", "d_ctx"))
            return {"score": m.forward(x["q"], x["d"], x["q_mask"], x["d_mask"])}

        def pin(r, tag=tag, ref=ref, qm=qm, dm=dm, gs=gs):
            q64, d64 = _leaf64(r["ctx"]["q_ctx"]), _leaf64(r["ctx"]["d_ctx"])
            w64, a64 = _leaf64(ref.kernel_bin_weights.weight.view(-1)), _leaf64(ref.kernel_alpha_scaler.view(-1))
            s, sec = O.kernel_pool_tk(q64, d64, qm.double(), dm.double(), ref.mu.view(-1).double(),
                                      ref.sigma.view(-1).double(), a64, w64)
            s.backward(gs.double())
            _pin(s.detach(), r["out"]["score"], f"tk[{tag}] score")
            _pin(q64.grad, r["gctx"]["q_ctx"], f"tk[{tag}] grad q_ctx")
            _pin(d64.grad, r["gctx"]["d_ctx"], f"tk[{tag}] grad d_ctx")
            _pin(w64.grad, r["gp"]["kernel_bin_weights.weight"].view(-1), f"tk[{tag}] grad kernel_bin_weights")
            _pin(a64.grad, r["gp"]["kernel_alpha_scaler"].view(-1), f"tk[{tag}] grad kernel_alpha_scaler")
            assert _floor_margin(sec["per_kernel_query"].detach(), qm, a64.detach()) > 1e-2

        _train_check_and_save(f"train_tk_{tag}", ref, inputs, ("q", "d"), forward, {"score": gs}, pin, lambda r: None,
                              extra={"cfg": np.array([emb, heads, layers, ff, max_len])})


def train_tk_sparse():
    torch.manual_seed(113)
    emb, heads, layers, proj, ff, max_len = 40, 4, 1, 16, 32, 64
    mu = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]
    ref = R.load_tk_sparse(emb, mu, [0.1] * 11, heads, layers, proj, ff, max_len, True)
    with torch.no_grad():
        ref.kernel_alpha_scaler.copy_(torch.rand_like(ref.kernel_alpha_scaler) + 0.5)
        ref.stop_word_reducer2.bias.fill_(0.3)     # so that relu() closes the gate for a share of the document terms
        ref.mixer.fill_(0.4)
        ref.mixer_stop.fill_(0.6)
    q, d, qm, dm = _tk_inputs(6, 12, 48, emb, seed=3400)
    gs, gstop = _seeded(3401, (q.shape[0],), (q.shape[0], 1, d.shape[1]))
    inputs = {"q": q, "d": d, "q_mask": qm, "d_mask": dm}
    pre_gate = {}

    def forward(m, x, retain):
        _wrap_representation(m, retain, ("q_ctx", "d_ctx"))
        h = m.stop_word_reducer2.register_forward_hook(lambda mod, i, o: pre_gate.__setitem__(o.dtype, o.detach()))
        score, stop = m.forward(x["q"], x["d"], x["q_mask"], x["d_mask"])
        h.remove()
        return {"score": score, "document_stop_words": retain("gate", stop)}

    def pin(r):
        q64, d64 = _leaf64(r["ctx"]["q_ctx"]), _leaf64(r["ctx"]["d_ctx"])
        g64 = _leaf64(r["ctx"]["gate"].squeeze(1))
        w64, a64 = _leaf64(ref.kernel_bin_weights.weight.view(-1)), _leaf64(ref.kernel_alpha_scaler.view(-1))
        s, sec = O.kernel_pool_tk_sparse(q64, d64, qm.double(), dm.double(), g64, ref.mu.view(-1).double(),
                                         ref.sigma.view(-1).double(), a64, w64)
        s.backward(gs.double())
        _pin(s.detach(), r["out"]["score"], "tk_sparse score")
        _pin(q64.grad, r["gctx"]["q_ctx"], "tk_sparse grad q_ctx")
        _pin(d64.grad, r["gctx"]["d_ctx"], "tk_sparse grad d_ctx")
        # the gate is also the second output: its gradient is the score's share plus the upstream gradient
        _pin(g64.grad + gstop.squeeze(1).double(), r["gctx"]["gate"].squeeze(1), "tk_sparse grad gate")
        _pin(w64.grad, r["gp"]["kernel_bin_weights.weight"].view(-1), "tk_sparse grad kernel_bin_weights")
        _pin(a64.grad, r["gp"]["kernel_alpha_scaler"].view(-1), "tk_sparse grad kernel_alpha_scaler")
        assert _floor_margin(sec["per_kernel_query"].detach(), qm, a64.detach()) > 1e-2

    def condition(r):
        gate = r["out"]["document_stop_words"].squeeze(1)
        closed = float((gate[dm.bool()] == 0).double().mean())
        assert 0.05 < closed < 0.95, f"the fixture should contain closed and open gates ({closed})"
        pre = pre_gate[torch.float64].squeeze(-1)[dm.bool()]
        assert float(pre.abs().min()) > 1e-4, "a gate's pre-activation sits at the relu kink"

    _train_check_and_save("train_tk_sparse", ref, inputs, ("q", "d"), forward,
                          {"score": gs, "document_stop_words": gstop}, pin, condition,
                          extra={"cfg": np.array([emb, heads, layers, proj, ff, max_len])})


def _tkl_second_best_gap(orig_score):
    """Smallest relative margin by which each of the greedy top-3 windows (sigir20_tkl.py:266-271) beats the best
    window still eligible at its step; windows at the -9900 sentinel (no live token) are exempt."""
    work = orig_score.clone()
    r = torch.arange(work.shape[1])
    gap = float("inf")
    for c in range(O.TKL_TOPK):
        top2 = torch.topk(work, 2, dim=1).values
        real = top2[:, 0] > -9900
        if real.any():
            rel = (top2[:, 0] - top2[:, 1]) / top2[:, 0].abs()
            gap = min(gap, float(rel[real].min().detach()))
        best = torch.argmax(work, dim=1)
        work[torch.abs(r - best.unsqueeze(-1)) < O.TKL_WINDOW / 2] = -10001 - c
    return gap


TKL_DATA_SEED = {"embedding": 3526, "log": 3511}   # seeds whose top-3 windows are clear of their runners-up


def train_tkl():
    emb, heads, layers, ff = 40, 4, 1, 32
    mu = [1.0, 0.9, 0.7, 0.5, 0.3, 0.1, -0.1, -0.3, -0.5, -0.7, -0.9]
    for sat in ("embedding", "log"):
        torch.manual_seed(114 if sat == "embedding" else 115)
        ref = R.load_tkl(emb, mu, [0.1] * 11, heads, layers, ff, 2000, True, True, sat)
        g = torch.Generator().manual_seed(3500)
        with torch.no_grad():   # well-conditioned saturation (the default bias 100 costs fp32 a 1e-3 share of the bar)
            ref.chunk_scoring.copy_(torch.rand(ref.chunk_scoring.shape, generator=g) + 0.5)
            ref.kernel_mult.copy_(torch.rand(ref.kernel_mult.shape, generator=g) + 0.5)
            ref.dense.weight.copy_(torch.randn(ref.dense.weight.shape, generator=g) * 0.1)
            ref.sat_emb_reduce1.weight.copy_(torch.randn(ref.sat_emb_reduce1.weight.shape, generator=g) * 0.3)
            ref.sat_normer.weight.copy_(torch.rand(2, generator=g) + 0.5)
            ref.sat_normer.bias.copy_(torch.randn(2, generator=g) * 0.1)
            for lin, scale, bias in ((ref.saturation_linear, 0.5, 3.0), (ref.saturation_linear2, 0.2, 2.0),
                                     (ref.saturation_linear3, 0.5, 1.0)):
                lin.weight.copy_(torch.randn(lin.weight.shape, generator=g) * scale)
                lin.bias.fill_(bias)
            ref.mixer.fill_(0.4)
        B, Lq, Ld = 3, 10, 120
        g = torch.Generator().manual_seed(TKL_DATA_SEED[sat])
        q = torch.randn(B, Lq, emb, generator=g) * 0.4
        d = torch.randn(B, Ld, emb, generator=g) * 0.4
        q_len = torch.tensor([10, 1, 4])
        d_len = torch.tensor([120, 90, 23])     # one document shorter than a chunk
        for b in range(B):  # exact matches
            d[b, 5] = q[b, 0]
            d[b, int(d_len[b]) - 3] = q[b, int(q_len[b]) - 1]
        qm = (torch.arange(Lq).unsqueeze(0) < q_len.unsqueeze(1)).float()
        dm = (torch.arange(Ld).unsqueeze(0) < d_len.unsqueeze(1)).float()
        q = q * qm.unsqueeze(-1)
        d = d * dm.unsqueeze(-1)
        (gs,) = _seeded(3501, (B,))
        inputs = {"q": q, "d": d, "q_mask": qm, "d_mask": dm}
        cd2, cp2, packed, pieces = O.tkl_chunk_documents(d, dm)
        chunk_mask = cp2[packed][:, O.TKL_OVERLAP:-O.TKL_OVERLAP].contiguous()
        secs, windows = {}, {}

        def forward(m, x, retain):
            _wrap_representation(m, retain, ("q_ctx", "doc_packed_ctx"))
            # the reference's window scores, dense(per_kernel) (sigir20_tkl.py:251): in "log" mode its secondary output
            # is unavailable (it reads `sat_influencer`, which only the "embedding" branch defines), so the top-3
            # windows are selected from these
            h = m.dense.register_forward_hook(lambda mod, i, o: windows.__setitem__(o.dtype, o.detach().squeeze(-1)))
            score, sec = (m.forward(x["q"], x["d"], x["q_mask"], x["d_mask"], output_secondary_output=True)
                          if sat == "embedding" else (m.forward(x["q"], x["d"], x["q_mask"], x["d_mask"]), None))
            h.remove()
            secs[score.dtype] = sec
            return {"score": score}

        def post(r):
            """The interaction stage reads the 40 centre rows of each packed 50-row chunk (sigir20_tkl.py:174): the
            overlap rows get no gradient from it, and only the centre rows are kept."""
            packed_ctx, g_packed = r["ctx"].pop("doc_packed_ctx"), r["gctx"].pop("doc_packed_ctx")
            assert (g_packed[:, :O.TKL_OVERLAP] == 0).all() and (g_packed[:, -O.TKL_OVERLAP:] == 0).all()
            r["ctx"]["doc_chunks_ctx"] = packed_ctx[:, O.TKL_OVERLAP:-O.TKL_OVERLAP]
            r["gctx"]["doc_chunks_ctx"] = g_packed[:, O.TKL_OVERLAP:-O.TKL_OVERLAP]

        def pin(r, sat=sat, ref=ref, qm=qm, gs=gs, packed=packed, pieces=pieces, chunk_mask=chunk_mask):
            q64 = _leaf64(r["ctx"]["q_ctx"])
            c64 = _leaf64(r["ctx"]["doc_chunks_ctx"])
            leaf = {"dense_weight": _leaf64(ref.dense.weight.view(-1)), "chunk_scoring": _leaf64(ref.chunk_scoring.view(-1)),
                    "sat_emb_reduce1_weight": _leaf64(ref.sat_emb_reduce1.weight.view(-1)),
                    "sat_normer_weight": _leaf64(ref.sat_normer.weight), "sat_normer_bias": _leaf64(ref.sat_normer.bias),
                    "kernel_mult0": _leaf64(ref.kernel_mult[0].reshape(-1))}
            for i in ("", "2", "3"):
                lin = getattr(ref, f"saturation_linear{i}")
                leaf[f"saturation_linear{i}_weight"] = _leaf64(lin.weight.view(-1))
                leaf[f"saturation_linear{i}_bias"] = _leaf64(lin.bias)
            params = dict(leaf, mu=ref.mu.detach().double(), sigma=ref.sigma.detach().double())
            s, sec = O.tkl_interaction(q64, qm.double(), c64, chunk_mask.double(), packed, pieces, params, sat)
            s.backward(gs.double())
            _pin(s.detach(), r["out"]["score"], f"tkl[{sat}] score")
            # the greedy top-3 (sigir20_tkl.py:254-271) on the reference's own window scores
            win = windows[torch.float64]
            if win.shape[1] < O.TKL_TOPK:
                win = torch.nn.functional.pad(win, (0, O.TKL_TOPK - win.shape[1]))
            win = win.masked_fill(win == 0, -9900)
            top_idx, _ = O.tkl_top_hills(win)
            assert torch.equal(top_idx, sec["top_non_overlapping_idx"]), "oracle and reference select other windows"
            if secs[torch.float64] is not None:
                assert torch.equal(top_idx, secs[torch.float64]["top_non_overlapping_idx"])
            r["top_idx"], r["windows"] = top_idx, win
            _pin(q64.grad, r["gctx"]["q_ctx"], f"tkl[{sat}] grad q_ctx")
            _pin(c64.grad, r["gctx"]["doc_chunks_ctx"], f"tkl[{sat}] grad doc_chunks_ctx")
            gp = r["gp"]
            _pin(leaf["dense_weight"].grad, gp["dense.weight"].view(-1), f"tkl[{sat}] grad dense.weight")
            _pin(leaf["chunk_scoring"].grad, gp["chunk_scoring"].view(-1), f"tkl[{sat}] grad chunk_scoring")
            if sat == "embedding":
                _pin(leaf["sat_emb_reduce1_weight"].grad, gp["sat_emb_reduce1.weight"].view(-1), "tkl grad sat_emb_reduce1")
                for n in ("sat_normer.weight", "sat_normer.bias", "saturation_linear.weight", "saturation_linear.bias",
                          "saturation_linear2.weight", "saturation_linear2.bias", "saturation_linear3.weight",
                          "saturation_linear3.bias"):
                    _pin(leaf[n.replace(".", "_")].grad, gp[n].view(-1), f"tkl grad {n}")
            else:
                _pin(leaf["kernel_mult0"].grad, gp["kernel_mult"][0].reshape(-1), "tkl[log] grad kernel_mult[0]")
                assert (gp["kernel_mult"][1:] == 0).all()

        def condition(r):
            gap = _tkl_second_best_gap(r["windows"])
            assert gap > 1e-3, f"a top-3 window beats its runner-up by only {gap:.2e} relative"

        # forward reads positional_features_q[:, :Lq] and positional_features_d[:, :50] only: the other rows are not stored
        _train_check_and_save(f"train_tkl_{sat}", ref, inputs, ("q", "d"), forward, {"score": gs}, pin, condition,
                              extra=lambda r, packed=packed, pieces=pieces, chunk_mask=chunk_mask: {
                                  "cfg": np.array([emb, heads, layers, ff]), "packed_indices": packed,
                                  "chunk_pieces": np.array(pieces), "doc_chunk_mask": chunk_mask,
                                  "top_non_overlapping_idx": r["top_idx"]},
                              trim={"positional_features_q": Lq, "positional_features_d": O.TKL_EXT}, post=post)


def train_colbert():
    """ColBERT.forward's masked pair scoring (colbert.py:68-75) on pass-through vectors, and the in-batch all-pairs
    scoring forward_inbatch_aggregation (:154-162) on the same vectors with n_q = n_d."""
    cls, inst = R.load_colbert()
    q, d, qm, dm = O.synth_colbert_inputs(6, 1, 8, 20, 32, seed=3600, dtype=torch.float32, full_q=False)
    qm[0, 1:] = 0
    q = q * qm.unsqueeze(-1)
    gs, gall = _seeded(3601, (6,), (6, 6))
    out, grads = {}, {}
    for dtype in (torch.float64, torch.float32):
        q_, d_ = q.to(dtype).clone().requires_grad_(True), d.to(dtype).clone().requires_grad_(True)
        s = inst.forward({"vecs": q_, "attention_mask": qm}, {"vecs": d_, "attention_mask": dm}, use_fp16=False)
        s.backward(gs.to(dtype))
        out[dtype, "score"], grads[dtype, "q"], grads[dtype, "d"] = s.detach(), q_.grad, d_.grad
        q_, d_ = q.to(dtype).clone().requires_grad_(True), d.to(dtype).clone().requires_grad_(True)
        a = cls.forward_inbatch_aggregation(inst, q_, qm, d_, dm)
        a.backward(gall.to(dtype))
        out[dtype, "allpairs"], grads[dtype, "ib_q"], grads[dtype, "ib_d"] = a.detach(), q_.grad, d_.grad
    print("train_colbert:")
    q64, d64 = _leaf64(q), _leaf64(d)
    s = O.maxsim_pairs(q64, d64, qm, dm)
    s.backward(gs.double())
    _pin(s.detach(), out[torch.float64, "score"], "colbert score")
    _pin(q64.grad, grads[torch.float64, "q"], "colbert grad q")
    _pin(d64.grad, grads[torch.float64, "d"], "colbert grad d")
    q64, d64 = _leaf64(q), _leaf64(d)
    a = O.maxsim_allpairs(q64, qm, d64, dm)
    a.backward(gall.double())
    _pin(a.detach(), out[torch.float64, "allpairs"], "colbert allpairs")
    _pin(q64.grad, grads[torch.float64, "ib_q"], "colbert in-batch grad q")
    _pin(d64.grad, grads[torch.float64, "ib_d"], "colbert in-batch grad d")
    # conditioning: the best document row of every live (pair, query term) beats the second best by > 1e-3 relative
    sc = torch.bmm(q.double(), d.double().transpose(1, 2)).masked_fill(~dm.bool().unsqueeze(1), -1000)
    allp = torch.einsum("aqe,bde->abqd", q.double(), d.double())
    allp = allp.masked_fill(~dm.bool().view(-1, 1, 1, dm.shape[1]), -1000)    # colbert.py:158's mask indexing
    for what, t, live in (("pairs", sc, qm.bool()), ("in-batch", allp, qm.bool().unsqueeze(1).expand(-1, 6, -1))):
        top2 = torch.topk(t, 2, dim=-1).values
        rel = ((top2[..., 0] - top2[..., 1]) / top2[..., 0].abs())[live]
        assert float(rel.min()) > 1e-3, f"colbert {what}: best and second-best document rows {float(rel.min()):.2e} apart"
    worst = max(_rel_err(v, out[torch.float64, k[1]]) for k, v in out.items() if k[0] == torch.float32)
    worst = max([worst] + [_rel_err(v, grads[torch.float64, k[1]]) for k, v in grads.items() if k[0] == torch.float32])
    assert worst <= FP32_SHARE, f"colbert: the fp32 reference run is {worst:.2e} off"
    print(f"  fp32 reference vs fp64: worst {worst:.2e}")
    for v in list(out.values()) + list(grads.values()):
        assert torch.isfinite(v).all()
    _save("train_colbert", q=q, d=d, q_mask=qm, d_mask=dm, gout__score=gs, gout__allpairs=gall,
          out__score=out[torch.float64, "score"].float(), out__allpairs=out[torch.float64, "allpairs"].float(),
          **{"gi__" + k: grads[torch.float64, k].float() for k in ("q", "d", "ib_q", "ib_d")})


def train_bert_dot():
    cls, inst = R.load_bert_dot()
    inst.train()
    qv, dv = _seeded(3700, (8, 64), (8, 64))
    (gs,) = _seeded(3701, (8,))
    res = {}
    for dtype in (torch.float64, torch.float32):
        q_, d_ = qv.to(dtype).clone().requires_grad_(True), dv.to(dtype).clone().requires_grad_(True)
        s = inst.forward({"vecs": q_}, {"vecs": d_}, use_fp16=False)
        s.backward(gs.to(dtype))
        res[dtype] = (s.detach(), q_.grad, d_.grad)
    print("train_bert_dot:")
    q64, d64 = _leaf64(qv), _leaf64(dv)
    s = O.dot_pairs(q64, d64)
    s.backward(gs.double())
    for got, want, what in zip((s.detach(), q64.grad, d64.grad), res[torch.float64], ("score", "grad qv", "grad dv")):
        _pin(got, want, f"bert_dot {what}")
    assert max(_rel_err(a, b) for a, b in zip(res[torch.float32], res[torch.float64])) <= FP32_SHARE
    _save("train_bert_dot", qv=qv, dv=dv, gout__score=gs, out__score=res[torch.float64][0].float(),
          gi__qv=res[torch.float64][1].float(), gi__dv=res[torch.float64][2].float())


TRAINING_FAMILIES = (("train_knrm", train_knrm), ("train_conv_knrm", train_conv_knrm), ("train_tk", train_tk),
                     ("train_tk_sparse", train_tk_sparse), ("train_tkl", train_tkl), ("train_colbert", train_colbert),
                     ("train_bert_dot", train_bert_dot))


def main():
    if not R.reference_available():
        print("reference not mounted at", R.REFERENCE_ROOT, "- cannot regenerate golden vectors", file=sys.stderr)
        return 1
    only = set(sys.argv[1:])   # e.g. `python -m oracle.make_golden knrm train_tk` regenerates two families
    for name, fn in (("knrm", golden_knrm), ("tk", golden_tk), ("tkl", golden_tkl), ("colbert", golden_colbert),
                     ("bert_dot", golden_bert_dot), ("tk_sparse", golden_tk_sparse), ("conv_knrm", golden_conv_knrm)):
        if not only or name in only:
            fn()
    for name, fn in TRAINING_FAMILIES:
        if not only or name in only:
            fn()
    return 0


if __name__ == "__main__":
    sys.exit(main())
