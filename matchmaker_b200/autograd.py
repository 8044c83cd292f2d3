"""torch.autograd bindings of the interaction kernels: forward and backward both run in
``libmatchmaker_b200.so``; autograd only routes tensors."""
from __future__ import annotations

from typing import Optional

import torch

from . import interaction


class _MaxSim(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, d, q_mask, d_mask, docs_per_query):
        # ctx.needs_input_grad follows the inputs' requires_grad, not the grad mode: it is all False for detached inputs
        # (nothing is saved then), but under torch.no_grad() inputs that require grad still take the argmax forward
        need_grad = ctx.needs_input_grad[0] or ctx.needs_input_grad[1]
        if need_grad:
            out, argmax = interaction.maxsim(q, d, q_mask, d_mask, docs_per_query=docs_per_query, return_argmax=True)
            ctx.save_for_backward(q, d, argmax)
            ctx.docs_per_query = docs_per_query
        else:
            out = interaction.maxsim(q, d, q_mask, d_mask, docs_per_query=docs_per_query)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        q, d, argmax = ctx.saved_tensors
        gq, gd = interaction.maxsim_bwd(q, d, grad_out, argmax, ctx.docs_per_query)
        return gq.to(q.dtype), gd.to(d.dtype), None, None, None


def maxsim(q: torch.Tensor, d: torch.Tensor, q_mask: Optional[torch.Tensor] = None,
           d_mask: Optional[torch.Tensor] = None, docs_per_query: int = 1) -> torch.Tensor:
    """Differentiable ColBERT max-sim (pairs mode); see :func:`matchmaker_b200.interaction.maxsim`."""
    return _MaxSim.apply(q, d, q_mask, d_mask, docs_per_query)


class _MaxSimAllPairs(torch.autograd.Function):
    """Only entered when a gradient is wanted (see maxsim_allpairs below): the argmax forward, then its backward."""

    @staticmethod
    def forward(ctx, q, q_mask, d, d_mask, reference_mask_indexing):
        out, argmax = interaction.maxsim_allpairs(q, q_mask, d, d_mask, reference_mask_indexing=reference_mask_indexing,
                                                  return_argmax=True)
        ctx.save_for_backward(q, d, argmax)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        q, d, argmax = ctx.saved_tensors
        gq, gd = interaction.maxsim_allpairs_bwd(q, d, grad_out, argmax)
        return (gq.to(q.dtype) if ctx.needs_input_grad[0] else None, None,
                gd.to(d.dtype) if ctx.needs_input_grad[2] else None, None, None)


def maxsim_allpairs(q: torch.Tensor, q_mask: Optional[torch.Tensor], d: torch.Tensor, d_mask: Optional[torch.Tensor],
                    reference_mask_indexing: bool = False) -> torch.Tensor:
    """Differentiable all-pairs max-sim [n_q, n_d] (in-batch negatives); see
    :func:`matchmaker_b200.interaction.maxsim_allpairs`.  The gradient follows the forward's argmax, so with
    ``reference_mask_indexing=True`` it is what autograd of colbert.py:154-162 gives, masks and all.

    Without a gradient to compute (grad mode off, e.g. under ``torch.no_grad()``, or neither q nor d requiring grad)
    this is exactly :func:`interaction.maxsim_allpairs`: no argmax, nothing saved, the inference kernels' bits.  The
    decision is taken here, outside the Function, because inside ``Function.forward`` grad mode is always off and
    ``ctx.needs_input_grad`` reflects only the inputs' ``requires_grad``."""
    if torch.is_grad_enabled() and (q.requires_grad or d.requires_grad):
        return _MaxSimAllPairs.apply(q, q_mask, d, d_mask, reference_mask_indexing)
    return interaction.maxsim_allpairs(q, q_mask, d, d_mask, reference_mask_indexing=reference_mask_indexing)


# "auto": forward that saves its cosines + tensor-core backward where the shape allows; "simt": always the FFMA backward
KP_TRAIN_IMPL = "auto"


class _KernelPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, d, q_mask, d_mask, mu, sigma, weight, alpha, log_scale, doc_gate, clamp_min, bias):
        # needs_input_grad (not tensor.requires_grad: parameters always require grad, also under no_grad)
        need_grad = any(ctx.needs_input_grad[i] for i in (0, 1, 6, 7, 9))
        # training step on the tensor cores when the shape allows it (KP_TRAIN_IMPL = "simt" keeps the FFMA backward)
        tc = (need_grad and KP_TRAIN_IMPL != "simt"
              and interaction.kernel_pool_train_supported(q.shape[1], d.shape[1], q.shape[2], mu.numel()))
        out = interaction.kernel_pool(q, d, q_mask, d_mask, mu, sigma, weight, alpha, log_scale,
                                      want_per_kernel=True, want_per_kernel_query=need_grad, doc_gate=doc_gate,
                                      clamp_min=clamp_min, bias=bias, save_for_backward=tc)
        if need_grad:
            empty = torch.empty(0, device=q.device)
            ctx.save_for_backward(q, d, q_mask, d_mask, mu, sigma, weight, alpha if alpha is not None else empty,
                                  out["per_kernel_query"], doc_gate if doc_gate is not None else empty,
                                  out["saved"] if tc else empty)
            ctx.tc = tc
            ctx.has_alpha, ctx.has_gate = alpha is not None, doc_gate is not None
            ctx.log_scale, ctx.clamp_min = log_scale, clamp_min
        ctx.mark_non_differentiable(out["per_kernel"])
        return out["score"], out["per_kernel"]

    @staticmethod
    def backward(ctx, grad_score, _grad_pk):
        q, d, q_mask, d_mask, mu, sigma, weight, alpha, S, gate, saved = ctx.saved_tensors
        alpha = alpha if ctx.has_alpha else None
        gate = gate if ctx.has_gate else None
        res = interaction.kernel_pool_bwd(q, d, q_mask, d_mask, mu, sigma, weight, alpha, S, grad_score, ctx.log_scale,
                                          doc_gate=gate, clamp_min=ctx.clamp_min, saved=saved if ctx.tc else None)
        gq, gd, ga, gw = res[:4]
        gg = res[4].view_as(gate) if gate is not None else None
        gw = gw.view_as(weight)
        ga = None if ga is None else ga.view_as(alpha)
        return gq.to(q.dtype), gd.to(d.dtype), None, None, None, None, gw, ga, None, gg, None, None


def kernel_pool(q, d, q_mask, d_mask, mu, sigma, weight, alpha=None, log_scale: float = 1.0, doc_gate=None,
                clamp_min: float = 1e-10, bias: float = 0.0):
    """Differentiable cosine + RBF kernel pooling: returns (score [B], per_kernel [B,K]); gradients flow to
    q, d, weight, alpha and doc_gate through the score (per_kernel is a detached by-product, as used by the
    reference's secondary outputs).  doc_gate / clamp_min / bias: see :func:`interaction.kernel_pool`."""
    return _KernelPool.apply(q, d, q_mask, d_mask, mu, sigma, weight, alpha, log_scale, doc_gate, clamp_min, bias)


class _DotPairs(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qv, dv):
        ctx.save_for_backward(qv, dv)
        return interaction.dot_pairs(qv, dv)

    @staticmethod
    def backward(ctx, g):
        qv, dv = ctx.saved_tensors
        # d<q,d>/dq = g*d, d/dd = g*q: a broadcast multiply on [B,dim] (not an interaction kernel)
        g = g.unsqueeze(-1)
        return (g * dv.float()).to(qv.dtype), (g * qv.float()).to(dv.dtype)


def dot_pairs(qv: torch.Tensor, dv: torch.Tensor) -> torch.Tensor:
    """Differentiable BERT_DOT pair score (bert_dot.py:62)."""
    return _DotPairs.apply(qv, dv)


class _TklInteraction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q_ctx, q_mask, doc_chunks, chunk_mask, packed, pieces, mu, sigma, dense_w, saturation, sat_params,
                sat_red_w, chunk_scoring):
        window = interaction.tkl_window_scores(q_ctx, q_mask, doc_chunks, chunk_mask, packed, pieces, mu, sigma, dense_w,
                                               saturation, sat_params, sat_red_w)
        score, orig, top_idx, top15 = interaction.tkl_top_hills(window, chunk_scoring)
        ctx.save_for_backward(q_ctx, q_mask, doc_chunks, chunk_mask, packed, mu, sigma, dense_w, sat_params,
                              sat_red_w if sat_red_w is not None else torch.empty(0, device=q_ctx.device),
                              chunk_scoring, top_idx, orig)
        ctx.pieces, ctx.saturation, ctx.has_red = pieces, saturation, sat_red_w is not None
        ctx.mark_non_differentiable(orig, top_idx, top15)
        return score, orig, top_idx, top15

    @staticmethod
    def backward(ctx, g_score, _g1, _g2, _g3):
        (q_ctx, q_mask, doc_chunks, chunk_mask, packed, mu, sigma, dense_w, sat_params, sat_red_w, chunk_scoring, top_idx,
         orig) = ctx.saved_tensors
        red = sat_red_w if ctx.has_red else None
        # the one-CTA-per-document kernel where its shared-memory plan fits, the feature-split one at BERT widths
        route = interaction.tkl_bwd_route(q_ctx.shape[1], q_ctx.shape[2], mu.numel())
        bwd = interaction.tkl_bwd_wide if route == "tkl_bwd_wide" else interaction.tkl_bwd
        gq, gc, g_dense, g_cs, g_sat, g_red = bwd(q_ctx, q_mask, doc_chunks, chunk_mask, packed, ctx.pieces,
                                                  mu, sigma, dense_w, ctx.saturation, sat_params, red, chunk_scoring,
                                                  top_idx, orig, g_score)
        return (gq.to(q_ctx.dtype), None, gc.to(doc_chunks.dtype), None, None, None, None, None, g_dense.view_as(dense_w),
                None, g_sat.view_as(sat_params), None if g_red is None else g_red.view_as(sat_red_w),
                g_cs.view_as(chunk_scoring))


def tkl_interaction(q_ctx, q_mask, doc_chunks, chunk_mask, packed, pieces, mu, sigma, dense_w, saturation, sat_params,
                    sat_red_w, chunk_scoring):
    """Differentiable TKL interaction stage (sigir20_tkl.py:180-286): returns (score [B], orig_score [B,W],
    top_idx [B,3], top15 [B,15]); gradients flow to q_ctx, doc_chunks, dense_w, sat_params, sat_red_w, chunk_scoring."""
    return _TklInteraction.apply(q_ctx, q_mask, doc_chunks, chunk_mask, packed, pieces, mu, sigma, dense_w, saturation,
                                 sat_params, sat_red_w, chunk_scoring)
