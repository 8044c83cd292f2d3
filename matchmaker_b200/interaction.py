"""Torch-facing wrappers of the interaction kernels (C ABI in ``include/matchmaker_b200.h``).

PyTorch is plumbing here: it owns device memory and the current stream; the arithmetic runs in
``libmatchmaker_b200.so``.  No function in this module has a CPU or eager-PyTorch fallback.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib

_DTYPES = {torch.float16: _lib.F16, torch.bfloat16: _lib.BF16, torch.float32: _lib.F32}
_MASK_DTYPES = {torch.bool: _lib.MASK_U8, torch.uint8: _lib.MASK_U8, torch.int32: _lib.MASK_I32,
                torch.int64: _lib.MASK_I64, torch.float32: _lib.MASK_F32}
# "tcgen05_ragged" is an alias of "tcgen05": the max-sim tensor-core kernel fetches only each document's live rows
# (up to its last unmasked one) whichever name selects it; the name stays accepted for existing callers.
_IMPLS = {"auto": _lib.IMPL_AUTO, "simt": _lib.IMPL_SIMT, "tcgen05": _lib.IMPL_TCGEN05,
          "tcgen05_docm": _lib.IMPL_TCGEN05_DOCM, "tcgen05_ragged": _lib.IMPL_TCGEN05_RAGGED}


def _require_cuda(*tensors: Optional[torch.Tensor]) -> torch.device:
    dev = None
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise _lib.MatchmakerB200Error(
                "matchmaker_b200 interaction ops run on CUDA (sm_90a) tensors only; got a "
                f"{t.device} tensor and there is no CPU fallback")
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise _lib.MatchmakerB200Error(f"tensors on different devices: {dev} vs {t.device}")
    return dev


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream(dev: torch.device) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


def _prep_mask(m: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    if m is None:
        return None
    if m.dtype not in _MASK_DTYPES:
        m = m != 0
    return m.contiguous()


def _common_mask_dtype(a: Optional[torch.Tensor], b: Optional[torch.Tensor]):
    """Both masks of one call share one element type (one `mask_dtype` argument)."""
    if a is not None and b is not None and a.dtype != b.dtype:
        a, b = (a != 0), (b != 0)
    code = _lib.MASK_NONE
    for m in (a, b):
        if m is not None:
            code = _MASK_DTYPES[m.dtype]
    return a, b, code


def maxsim(q: torch.Tensor, d: torch.Tensor, q_mask: Optional[torch.Tensor] = None,
           d_mask: Optional[torch.Tensor] = None, docs_per_query: int = 1,
           pair_q: Optional[torch.Tensor] = None, pair_d: Optional[torch.Tensor] = None,
           impl: str = "auto", return_argmax: bool = False, pair_dmask: Optional[torch.Tensor] = None):
    """ColBERT max-sim scores, fp32.

    q [n_q, Lq, dim], d [n_d, Ld, dim] (fp16 / bf16 / fp32, same dtype), masks [n, L] (nonzero =
    token).  Pair p scores query ``pair_q[p]`` (default ``p // docs_per_query``) against document
    ``pair_d[p]`` (default ``p``).  Semantics: matchmaker/models/colbert.py:68-75 / :100-112.
    """
    dev = _require_cuda(q, d, q_mask, d_mask, pair_q, pair_d, pair_dmask)
    if q.dtype != d.dtype or q.dtype not in _DTYPES:
        raise _lib.MatchmakerB200Error(f"q/d must share a dtype in fp16/bf16/fp32, got {q.dtype}, {d.dtype}")
    if q.dim() != 3 or d.dim() != 3 or q.shape[-1] != d.shape[-1]:
        raise _lib.MatchmakerB200Error(f"expected q [n_q,Lq,dim], d [n_d,Ld,dim]; got {tuple(q.shape)}, {tuple(d.shape)}")
    q = q.contiguous()
    d = d.contiguous()
    q_mask, d_mask, mcode = _common_mask_dtype(_prep_mask(q_mask), _prep_mask(d_mask))
    n_q, Lq, dim = q.shape
    n_d, Ld, _ = d.shape
    if q_mask is not None and tuple(q_mask.shape) != (n_q, Lq):
        raise _lib.MatchmakerB200Error("q_mask shape mismatch")
    if d_mask is not None and tuple(d_mask.shape) != (n_d, Ld):
        raise _lib.MatchmakerB200Error("d_mask shape mismatch")
    if pair_q is not None or pair_d is not None:
        if pair_q is None or pair_d is None:
            raise _lib.MatchmakerB200Error("pair_q and pair_d must be given together")
        pair_q = pair_q.to(torch.int32).contiguous()
        pair_d = pair_d.to(torch.int32).contiguous()
        n_pairs = pair_q.numel()
        if pair_d.numel() != n_pairs:
            raise _lib.MatchmakerB200Error("pair_q / pair_d length mismatch")
        if pair_dmask is not None:
            pair_dmask = pair_dmask.to(torch.int32).contiguous()
            if pair_dmask.numel() != n_pairs:
                raise _lib.MatchmakerB200Error("pair_dmask length mismatch")
    else:
        n_pairs = n_d
        if n_q * docs_per_query < n_d:
            raise _lib.MatchmakerB200Error("n_q * docs_per_query < n_d")
    out = torch.empty(n_pairs, dtype=torch.float32, device=dev)
    argmax = torch.empty((n_pairs, Lq), dtype=torch.int32, device=dev) if return_argmax else None
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_maxsim_fwd(_ptr(q), _ptr(d), _ptr(q_mask), _ptr(d_mask), _ptr(pair_q), _ptr(pair_d),
                                   _ptr(pair_dmask), _ptr(out), _ptr(argmax), n_q, n_d, n_pairs, docs_per_query, Lq, Ld, dim,
                                   _DTYPES[q.dtype], mcode, _IMPLS[impl], _stream(dev))
    _lib.check(rc, "mmb200_maxsim_fwd")
    return (out, argmax) if return_argmax else out


def maxsim_allpairs(q: torch.Tensor, q_mask: Optional[torch.Tensor], d: torch.Tensor,
                    d_mask: Optional[torch.Tensor], impl: str = "auto",
                    reference_mask_indexing: bool = False, return_argmax: bool = False):
    """All query x document max-sim scores [n_q, n_d] (colbert.py:154-162).

    ``reference_mask_indexing=True`` reproduces the reference bit-for-bit: colbert.py:158 expands
    ``document_mask`` [n_d, Ld] along the *query* axis of the [n_q, n_d, Lq, Ld] score tensor, i.e. pair
    (a, b) is masked with the mask of document ``a`` (only defined for n_q == n_d, the in-batch case).
    The default applies each document's own mask.  ``return_argmax=True`` also returns the argmax
    [n_q * n_d, Lq] int32 of pair a * n_d + b, what :func:`maxsim_allpairs_bwd` takes."""
    n_q, n_d = q.shape[0], d.shape[0]
    idx = torch.arange(n_q * n_d, device=q.device, dtype=torch.int32)
    pq = torch.div(idx, n_d, rounding_mode="floor").to(torch.int32)
    pd = (idx - pq * n_d).to(torch.int32)
    pdm = None
    if reference_mask_indexing and d_mask is not None:
        if n_q != n_d:
            raise _lib.MatchmakerB200Error("reference mask indexing (colbert.py:158) needs n_q == n_d")
        pdm = pq
    res = maxsim(q, d, q_mask, d_mask, pair_q=pq, pair_d=pd, impl=impl, pair_dmask=pdm, return_argmax=return_argmax)
    if return_argmax:
        return res[0].view(n_q, n_d), res[1]
    return res.view(n_q, n_d)


def maxsim_allpairs_bwd(q: torch.Tensor, d: torch.Tensor, grad_out: torch.Tensor,
                        argmax: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Gradients of :func:`maxsim_allpairs` w.r.t. q [n_q, Lq, dim] and d [n_d, Ld, dim], fp32, from
    grad_out [n_q, n_d] and the forward's argmax [n_q * n_d, Lq] (either mask indexing: the gradient
    follows the argmax)."""
    dev = _require_cuda(q, d, grad_out, argmax)
    if q.dtype != d.dtype or q.dtype not in _DTYPES:
        raise _lib.MatchmakerB200Error(f"q/d must share a dtype in fp16/bf16/fp32, got {q.dtype}, {d.dtype}")
    if q.dim() != 3 or d.dim() != 3 or q.shape[-1] != d.shape[-1]:
        raise _lib.MatchmakerB200Error(f"expected q [n_q,Lq,dim], d [n_d,Ld,dim]; got {tuple(q.shape)}, {tuple(d.shape)}")
    q = q.contiguous()
    d = d.contiguous()
    n_q, Lq, dim = q.shape
    n_d, Ld, _ = d.shape
    if grad_out.numel() != n_q * n_d:
        raise _lib.MatchmakerB200Error(f"grad_out has {grad_out.numel()} elements, expected n_q * n_d = {n_q * n_d}")
    if argmax.dtype != torch.int32 or tuple(argmax.shape) != (n_q * n_d, Lq):
        raise _lib.MatchmakerB200Error(f"argmax must be int32 [{n_q * n_d}, {Lq}], got {argmax.dtype} "
                                       f"{tuple(argmax.shape)}")
    grad_out = grad_out.to(torch.float32).contiguous()
    gq = torch.empty((n_q, Lq, dim), dtype=torch.float32, device=dev)
    gd = torch.empty((n_d, Ld, dim), dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_maxsim_allpairs_bwd(_ptr(q), _ptr(d), _ptr(grad_out), _ptr(argmax.contiguous()), _ptr(gq),
                                            _ptr(gd), n_q, n_d, Lq, Ld, dim, _DTYPES[q.dtype], _stream(dev))
    _lib.check(rc, "mmb200_maxsim_allpairs_bwd")
    return gq, gd


def maxsim_bwd(q: torch.Tensor, d: torch.Tensor, grad_out: torch.Tensor, argmax: torch.Tensor,
               docs_per_query: int = 1) -> Tuple[torch.Tensor, torch.Tensor]:
    """Gradients of :func:`maxsim` (pairs mode) w.r.t. q and d, fp32."""
    dev = _require_cuda(q, d, grad_out, argmax)
    q = q.contiguous()
    d = d.contiguous()
    n_q, Lq, dim = q.shape
    n_d, Ld, _ = d.shape
    grad_out = grad_out.to(torch.float32).contiguous()
    gq = torch.empty((n_q, Lq, dim), dtype=torch.float32, device=dev)
    gd = torch.empty((n_d, Ld, dim), dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_maxsim_bwd(_ptr(q), _ptr(d), _ptr(grad_out), _ptr(argmax.contiguous()), _ptr(gq), _ptr(gd),
                                   n_q, n_d, n_d, docs_per_query, Lq, Ld, dim, _DTYPES[q.dtype], _stream(dev))
    _lib.check(rc, "mmb200_maxsim_bwd")
    return gq, gd


def maxsim_host(q: torch.Tensor, d: torch.Tensor, q_mask: Optional[torch.Tensor] = None,
                d_mask: Optional[torch.Tensor] = None, docs_per_query: int = 1, chunk_pairs: int = 0,
                device: Optional[torch.device] = None) -> torch.Tensor:
    """End-to-end max-sim over HOST tensors (pinned for full PCIe rate): document slabs are streamed to the
    GPU and scored while the next slab is in flight; returns a host fp32 tensor.  This is the call
    dense_retrieval.py:398-412 would make for token matrices gathered from the CPU memmap storage."""
    for t in (q, d, q_mask, d_mask):
        if t is not None and t.is_cuda:
            raise _lib.MatchmakerB200Error("maxsim_host takes host tensors; use maxsim() for device tensors")
    if q.dtype != d.dtype or q.dtype not in _DTYPES:
        raise _lib.MatchmakerB200Error("q/d must share a dtype in fp16/bf16/fp32")
    q = q.contiguous()
    d = d.contiguous()
    q_mask, d_mask, mcode = _common_mask_dtype(_prep_mask(q_mask), _prep_mask(d_mask))
    n_q, Lq, dim = q.shape
    n_d, Ld, _ = d.shape
    if n_q * docs_per_query < n_d:
        raise _lib.MatchmakerB200Error("n_q * docs_per_query < n_d")
    out = torch.empty(n_d, dtype=torch.float32, pin_memory=True)
    lib = _lib.load()
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    with torch.cuda.device(dev):
        rc = lib.mmb200_maxsim_fwd_host(_ptr(q), _ptr(d), _ptr(q_mask), _ptr(d_mask), _ptr(out), n_q, n_d,
                                        docs_per_query, Lq, Ld, dim, _DTYPES[q.dtype], mcode, chunk_pairs)
    _lib.check(rc, "mmb200_maxsim_fwd_host")
    return out


def _f32c(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).contiguous()


def kernel_pool(q: torch.Tensor, d: torch.Tensor, q_mask: torch.Tensor, d_mask: torch.Tensor,
                mu: torch.Tensor, sigma: torch.Tensor, weight: torch.Tensor, alpha: Optional[torch.Tensor] = None,
                log_scale: float = 1.0, want_per_kernel: bool = False, want_per_kernel_query: bool = False,
                want_cosine: bool = False, impl: str = "auto", doc_gate: Optional[torch.Tensor] = None,
                clamp_min: float = 1e-10, bias: float = 0.0, save_for_backward: bool = False):
    """Cosine match matrix + RBF kernel pooling, forward (knrm.py:52-84 / ecai20_tk.py:105-124).

    q [B,Lq,D], d [B,Ld,D] fp32; masks [B,L]; mu/sigma/weight(/alpha) [K].  Returns a dict with "score"
    [B] and, on request, "per_kernel" [B,K], "per_kernel_query" [B,Lq,K], "cosine" [B,Lq,Ld].

    Variants: ``doc_gate`` [B,Ld] multiplies every activation of its document term (TK-Sparse,
    cikm20_tk_sparse.py:135); ``clamp_min`` / ``bias`` are the 1e-4 floor and the Linear bias of IDCM's ESM scorer
    (sigir21_idcm.py:185-186).

    ``save_for_backward=True`` (shapes for which :func:`kernel_pool_train_supported` holds) runs the
    training forward: the result additionally carries "saved", the opaque state the tensor-core backward consumes
    (:func:`kernel_pool_bwd` with ``saved=``), and "per_kernel_query"."""
    dev = _require_cuda(q, d, q_mask, d_mask, mu, sigma, weight, alpha, doc_gate)
    if q.dtype != torch.float32 or d.dtype != torch.float32:
        q, d = q.float(), d.float()  # the reference runs TK/KNRM with use_fp16: False (tk.yaml:6)
    q, d = q.contiguous(), d.contiguous()
    B, Lq, D = q.shape
    _, Ld, _ = d.shape
    if d.shape[0] != B or d.shape[2] != D:
        raise _lib.MatchmakerB200Error(f"shape mismatch: q {tuple(q.shape)} d {tuple(d.shape)}")
    q_mask, d_mask, mcode = _common_mask_dtype(_prep_mask(q_mask), _prep_mask(d_mask))
    mu, sigma, weight = _f32c(mu).view(-1), _f32c(sigma).view(-1), _f32c(weight).view(-1)
    alpha = None if alpha is None else _f32c(alpha).view(-1)
    K = mu.numel()
    score = torch.empty(B, dtype=torch.float32, device=dev)
    pk = torch.empty((B, K), dtype=torch.float32, device=dev) if want_per_kernel else None
    pkq = torch.empty((B, Lq, K), dtype=torch.float32, device=dev) if want_per_kernel_query else None
    cos = torch.empty((B, Lq, Ld), dtype=torch.float32, device=dev) if want_cosine else None
    gate = None
    if doc_gate is not None:
        gate = _f32c(doc_gate).reshape(B, Ld)
    lib = _lib.load()
    if save_for_backward:
        if want_cosine or not kernel_pool_train_supported(Lq, Ld, D, K):
            raise _lib.MatchmakerB200Error("kernel_pool(save_for_backward=True): outside the tensor-core training envelope")
        if pkq is None:
            pkq = torch.empty((B, Lq, K), dtype=torch.float32, device=dev)
        saved = torch.empty(int(lib.mmb200_kernel_pool_saved_floats(B, Ld)), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            rc = lib.mmb200_kernel_pool_fwd_train(_ptr(q), _ptr(d), _ptr(q_mask), _ptr(d_mask), _ptr(gate), _ptr(mu), _ptr(sigma),
                                                  _ptr(alpha), _ptr(weight), _ptr(score), _ptr(pk), _ptr(pkq), _ptr(saved),
                                                  B, Lq, Ld, D, K, float(log_scale), float(clamp_min), float(bias), mcode,
                                                  _stream(dev))
        _lib.check(rc, "mmb200_kernel_pool_fwd_train")
        return {"score": score, "per_kernel": pk, "per_kernel_query": pkq, "cosine": None, "saved": saved}
    with torch.cuda.device(dev):
        rc = lib.mmb200_kernel_pool_fwd_ex(_ptr(q), _ptr(d), _ptr(q_mask), _ptr(d_mask), _ptr(gate), _ptr(mu), _ptr(sigma),
                                           _ptr(alpha), _ptr(weight), _ptr(score), _ptr(pk), _ptr(pkq), _ptr(cos),
                                           B, Lq, Ld, D, K, float(log_scale), float(clamp_min), float(bias), mcode,
                                           _IMPLS[impl], _stream(dev))
    _lib.check(rc, "mmb200_kernel_pool_fwd_ex")
    return {"score": score, "per_kernel": pk, "per_kernel_query": pkq, "cosine": cos}


def kernel_pool_train_supported(Lq: int, Ld: int, D: int, K: int) -> bool:
    """True when the tensor-core training pair (forward that saves its cosines + tensor-core backward) covers the shape."""
    return bool(_lib.load().mmb200_kernel_pool_train_tc_supported(int(Lq), int(Ld), int(D), int(K)))


def kernel_pool_bwd(q, d, q_mask, d_mask, mu, sigma, weight, alpha, per_kernel_query, grad_score,
                    log_scale: float = 1.0, doc_gate: Optional[torch.Tensor] = None, clamp_min: float = 1e-10,
                    saved: Optional[torch.Tensor] = None):
    """Backward of :func:`kernel_pool`: returns (grad_q, grad_d, grad_alpha or None, grad_weight[, grad_gate when a
    ``doc_gate`` was given]).  With ``saved`` (from ``kernel_pool(save_for_backward=True)``) both contractions run on the
    tensor cores (tf32 operands: gradients within a few 1e-4 relative of the fp32 expression)."""
    dev = _require_cuda(q, d, per_kernel_query, grad_score)
    q, d = q.float().contiguous(), d.float().contiguous()
    B, Lq, D = q.shape
    Ld = d.shape[1]
    q_mask, d_mask, mcode = _common_mask_dtype(_prep_mask(q_mask), _prep_mask(d_mask))
    mu, sigma, weight = _f32c(mu).view(-1), _f32c(sigma).view(-1), _f32c(weight).view(-1)
    alpha_c = None if alpha is None else _f32c(alpha).view(-1)
    K = mu.numel()
    gq = torch.empty_like(q)
    gd = torch.empty_like(d)
    ga = torch.empty(K, dtype=torch.float32, device=dev)
    gw = torch.empty(K, dtype=torch.float32, device=dev)
    ws = torch.empty(2 * B * K, dtype=torch.float32, device=dev)
    gate = None if doc_gate is None else _f32c(doc_gate).reshape(B, Ld)
    gg = None if doc_gate is None else torch.empty((B, Ld), dtype=torch.float32, device=dev)
    lib = _lib.load()
    if saved is not None:
        with torch.cuda.device(dev):
            rc = lib.mmb200_kernel_pool_bwd_saved(_ptr(q), _ptr(d), _ptr(q_mask), _ptr(d_mask), _ptr(gate), _ptr(mu), _ptr(sigma),
                                                  _ptr(alpha_c), _ptr(weight), _ptr(per_kernel_query.contiguous()),
                                                  _ptr(saved), _ptr(_f32c(grad_score)), _ptr(gq), _ptr(gd), _ptr(gg), _ptr(ga),
                                                  _ptr(gw), _ptr(ws), B, Lq, Ld, D, K, float(log_scale), float(clamp_min),
                                                  mcode, _stream(dev))
        _lib.check(rc, "mmb200_kernel_pool_bwd_saved")
        if doc_gate is not None:
            return gq, gd, (ga if alpha is not None else None), gw, gg
        return gq, gd, (ga if alpha is not None else None), gw
    with torch.cuda.device(dev):
        rc = lib.mmb200_kernel_pool_bwd_ex(_ptr(q), _ptr(d), _ptr(q_mask), _ptr(d_mask), _ptr(gate), _ptr(mu), _ptr(sigma),
                                           _ptr(alpha_c), _ptr(weight), _ptr(per_kernel_query.contiguous()),
                                           _ptr(_f32c(grad_score)), _ptr(gq), _ptr(gd), _ptr(gg), _ptr(ga), _ptr(gw),
                                           _ptr(ws), B, Lq, Ld, D, K, float(log_scale), float(clamp_min), mcode,
                                           _stream(dev))
    _lib.check(rc, "mmb200_kernel_pool_bwd_ex")
    if doc_gate is not None:
        return gq, gd, (ga if alpha is not None else None), gw, gg
    return gq, gd, (ga if alpha is not None else None), gw


def dot_pairs(qv: torch.Tensor, dv: torch.Tensor) -> torch.Tensor:
    """score[b] = <qv[b], dv[b]> in fp32 (bert_dot.py:62).  qv, dv [B, dim], same dtype."""
    dev = _require_cuda(qv, dv)
    if qv.dtype != dv.dtype or qv.dtype not in _DTYPES or qv.shape != dv.shape or qv.dim() != 2:
        raise _lib.MatchmakerB200Error(f"dot_pairs expects two [B,dim] tensors of one dtype, got {tuple(qv.shape)} "
                                       f"{qv.dtype} / {tuple(dv.shape)} {dv.dtype}")
    qv, dv = qv.contiguous(), dv.contiguous()
    out = torch.empty(qv.shape[0], dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_dot_pairs(_ptr(qv), _ptr(dv), _ptr(out), qv.shape[0], qv.shape[1], _DTYPES[qv.dtype],
                                  _stream(dev))
    _lib.check(rc, "mmb200_dot_pairs")
    return out


TKL_CHUNK, TKL_WINDOW = 40, 30
_TKL_COVER_CACHE = {}


def tkl_kernel_set_covers(mu: torch.Tensor, sigma: torch.Tensor) -> bool:
    """True when every cosine in [-1, 1] activates at least one RBF kernel under ex2.approx.ftz, i.e. when the window
    token count of sigir20_tkl.py:210 equals the count of unmasked positions (tkl_ts.cu explains why that matters).
    Same sweep as the device-side plan kernel; evaluated on the host once per (mu, sigma) tensor version -- they are
    constant buffers of the model -- so that the launch path knows which kernel to enqueue without a device round trip."""
    key = (mu.data_ptr(), mu._version, sigma.data_ptr(), sigma._version, mu.numel())
    hit = _TKL_COVER_CACHE.get(key)
    if hit is not None:
        return hit
    m, sg = mu.detach().float().view(-1).cpu().tolist(), sigma.detach().float().view(-1).cpu().tolist()
    x, ok = -1.01, True
    while x < 1.01:
        reach = x
        for mk, sk in zip(m, sg):
            h = 11.0 * sk / (0.5 * 1.4426950408889634) ** 0.5
            if mk - h <= x and mk + h > reach:
                reach = mk + h
        if reach <= x:
            ok = False
            break
        x = reach
    if len(_TKL_COVER_CACHE) > 64:
        _TKL_COVER_CACHE.clear()
    _TKL_COVER_CACHE[key] = ok
    return ok


def tkl_window_scores(q_ctx: torch.Tensor, q_mask: torch.Tensor, doc_chunks: torch.Tensor, chunk_mask: torch.Tensor,
                      packed_indices: torch.Tensor, chunk_pieces: int, mu: torch.Tensor, sigma: torch.Tensor,
                      dense_weight: torch.Tensor, saturation: str, sat_params: torch.Tensor,
                      sat_red_weight: Optional[torch.Tensor] = None, impl: str = "auto") -> torch.Tensor:
    """Window scores [B, W] of the TKL interaction stage (sigir20_tkl.py:180-252).

    ``packed_indices`` [B*C] bool is the reference's chunk packing mask (:159); ``doc_chunks`` [Nc,40,D] /
    ``chunk_mask`` [Nc,40] are the packed, contextualised chunks without overlap (:174-175)."""
    dev = _require_cuda(q_ctx, q_mask, doc_chunks, chunk_mask, packed_indices, mu, sigma, dense_weight, sat_params)
    q_ctx = q_ctx.float().contiguous()
    doc_chunks = doc_chunks.float().contiguous()
    B, Lq, D = q_ctx.shape
    C = int(chunk_pieces)
    if packed_indices.numel() != B * C or doc_chunks.shape[1] != TKL_CHUNK:
        raise _lib.MatchmakerB200Error("tkl_window_scores: inconsistent chunk packing")
    slot_to_packed = _tkl_slot_map(packed_indices)
    q_mask, chunk_mask, mcode = _common_mask_dtype(_prep_mask(q_mask), _prep_mask(chunk_mask))
    mu, sigma, dense_weight = _f32c(mu).view(-1), _f32c(sigma).view(-1), _f32c(dense_weight).view(-1)
    sat_params = _f32c(sat_params).view(-1)
    sat_code = {"embedding": 0, "log": 1}[saturation]
    red = None if sat_red_weight is None else _f32c(sat_red_weight).view(-1)
    K = mu.numel()
    W = (C * TKL_CHUNK - TKL_WINDOW) // 2 + 1
    out = torch.empty((B, W), dtype=torch.float32, device=dev)
    if impl == "auto":
        # decide on the host (cached per parameter version) so that only ONE of the two kernels is enqueued; the library's
        # own device-side check stays in force (a forced tensor-core call on a kernel set without cover writes zeros)
        impl = "tcgen05" if (Lq * K <= 512 and K <= 16 and tkl_kernel_set_covers(mu, sigma)) else "simt"
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_tkl_window_scores(_ptr(q_ctx), _ptr(q_mask), _ptr(doc_chunks), _ptr(chunk_mask),
                                          _ptr(slot_to_packed), _ptr(mu), _ptr(sigma), _ptr(dense_weight), _ptr(red),
                                          _ptr(sat_params), _ptr(out), B, doc_chunks.shape[0], Lq, D, C, K, sat_code, mcode,
                                          _IMPLS[impl], _stream(dev))
    _lib.check(rc, "mmb200_tkl_window_scores")
    return out


def tkl_top_hills(window_score: torch.Tensor, chunk_scoring: torch.Tensor):
    """Greedy top-3 windows with +-15 suppression, +-1/+-2 neighbours, weighted sum (sigir20_tkl.py:254-286).
    Returns (score [B], orig_score [B,W], top_idx [B,3] int64, top15 [B,15]); ``window_score`` is not modified."""
    dev = _require_cuda(window_score, chunk_scoring)
    ws = window_score.float().contiguous()
    B, W = ws.shape
    orig = torch.empty_like(ws)
    top_idx = torch.empty((B, 3), dtype=torch.int64, device=dev)
    top15 = torch.empty((B, 15), dtype=torch.float32, device=dev)
    score = torch.empty(B, dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_tkl_top_hills(_ptr(ws), _ptr(orig), _ptr(_f32c(chunk_scoring).view(-1)), _ptr(top_idx), _ptr(top15),
                                      _ptr(score), B, W, _stream(dev))
    _lib.check(rc, "mmb200_tkl_top_hills")
    return score, orig, top_idx, top15


FLAT_IP_MAX_K = 1024


def flat_ip_split_f32(x: torch.Tensor, role: str, scale_log2: Optional[int] = None) -> Tuple[torch.Tensor, int]:
    """fp32 vectors -> the fp16 hi / lo layout of MMB200_F32_SPLIT16: x * 2^s = hi + lo (+ a 2^-22 relative residue),
    s chosen so that the largest magnitude sits just below 2^15 (fp16 range, lo halves stay normal numbers).
    role "passages": [n, 2*dim] = [hi | lo] (the index stores this once); role "queries": [nq, 3*dim] = [hi | lo | hi].
    Returns (split tensor, s).  Elementwise format conversion, not scoring arithmetic."""
    import math
    x = x.float()
    if scale_log2 is None:
        amax = float(x.abs().max().item()) if x.numel() else 0.0
        scale_log2 = int(math.floor(math.log2(32000.0 / amax))) if (amax > 0.0 and math.isfinite(amax)) else 0
    xs = torch.ldexp(x, torch.tensor(scale_log2, device=x.device))
    hi = xs.to(torch.float16)
    lo = (xs - hi.float()).to(torch.float16)
    parts = [hi, lo] if role == "passages" else [hi, lo, hi]
    return torch.cat(parts, dim=1).contiguous(), scale_log2


FP8_MAX = 448.0   # largest finite torch.float8_e4m3fn value


def fp8_scale_log2(amax: torch.Tensor) -> torch.Tensor:
    """The E4M3 scale rule, elementwise: the largest integer s with amax * 2^s <= 448 (int32), 0 where amax is 0.
    Exact: with amax = m * 2^e (0.5 <= m < 1), s = 9 - e when m <= 0.875 and 8 - e otherwise.  Runs on the tensor's
    device without a host synchronisation (the per-query scales of a search); a non-finite amax gives a meaningless
    s, so callers that must refuse one check it (:func:`fp8_store_scale`)."""
    m, e = torch.frexp(amax.float())
    s = torch.where(m <= 0.875, 9 - e, 8 - e)
    return torch.where(amax > 0, s, torch.zeros_like(s)).to(torch.int32)


def fp8_store_scale(amax: float) -> int:
    """The E4M3 scale rule for one host value (a store's largest |x|); raises on a non-finite or negative amax."""
    import math
    if not math.isfinite(amax) or amax < 0:
        raise _lib.MatchmakerB200Error(f"fp8 store scale: the largest |x| of the rows is {amax}, not a finite value")
    return int(fp8_scale_log2(torch.tensor([amax], dtype=torch.float32))[0])


def _pow2_f32(e: torch.Tensor) -> torch.Tensor:
    """2^e as fp32 for integer e in [-126, 127], built from the exponent bits (exact)."""
    return ((e.to(torch.int32) + 127) << 23).view(torch.float32)


def fp8_quantize(x: torch.Tensor, scale_log2) -> torch.Tensor:
    """e4m3_rn(x * 2^s) as torch.float8_e4m3fn: torch's cast of the fp32 value x * 2^s.  scale_log2 is an int or an
    integer tensor over the leading dimensions of x (one scale per query of a [N, Lq, dim] batch).  The product is
    taken as two power-of-two factors, so it is exact for every s the scale rule gives.  Elementwise format
    conversion, not scoring arithmetic."""
    s = torch.as_tensor(scale_log2, dtype=torch.int32, device=x.device)
    while s.dim() < x.dim():
        s = s.unsqueeze(-1)
    h = torch.div(s, 2, rounding_mode="floor")
    y = x.to(torch.float32, copy=True)
    y.mul_(_pow2_f32(h)).mul_(_pow2_f32(s - h))
    return y.to(torch.float8_e4m3fn)


def fp8_unscale(scores: torch.Tensor, scale_log2: torch.Tensor) -> torch.Tensor:
    """scores * 2^-scale_log2 (an integer tensor over the leading dimensions of scores), exact, in fp32; void scores
    (-inf, -3.4028235e38) are left as they are."""
    e = scale_log2.to(torch.float64)
    while e.dim() < scores.dim():
        e = e.unsqueeze(-1)
    out = (scores.double() * torch.exp2(-e)).float()
    return torch.where(scores > -3.0e38, out, scores)


def _fp8_pair(a: torch.Tensor, b: torch.Tensor, what: str) -> bool:
    """True when both operands are e4m3; raises when only one is."""
    fa, fb = a.dtype == torch.float8_e4m3fn, b.dtype == torch.float8_e4m3fn
    if fa != fb:
        raise _lib.MatchmakerB200Error(f"{what}: e4m3 needs both operands in torch.float8_e4m3fn, got {a.dtype}, "
                                       f"{b.dtype}")
    return fa


def flat_ip_topk(queries: torch.Tensor, passages: torch.Tensor, k: int, ids: Optional[torch.Tensor] = None,
                 id_base: int = 0, split_scale: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exact inner-product top-k of every query against a resident passage shard (faiss IndexFlatIP
    semantics, faiss_indices.py:34).  queries [nq,dim], passages [n,dim] fp16/bf16; returns
    (scores [nq,k] f32 descending, ids [nq,k] int64); ties by id ascending.  1 <= k <= 1024.

    fp32 storage (``token_dtype: float32``): pass ``passages`` = flat_ip_split_f32(p, "passages")[0] ([n, 2*dim] fp16)
    together with its scale as ``split_scale``; queries (fp32 [nq, dim]) are split here, scores are returned unscaled.

    E4M3 (both operands torch.float8_e4m3fn, dim % 128 == 0, 128 <= dim <= 1024): the scores are the sums of products
    of the stored values, i.e. in the scaled domain of :func:`fp8_quantize`; the caller unscales."""
    dev = _require_cuda(queries, passages, ids)
    fp8 = _fp8_pair(queries, passages, "flat_ip_topk")
    if not fp8 and passages.dtype not in (torch.float16, torch.bfloat16):
        raise _lib.MatchmakerB200Error("flat_ip_topk: passage storage must be fp16 / bf16, or the fp16 split of fp32 "
                                       "(flat_ip_split_f32)")
    n = passages.shape[0]
    unscale = None
    if split_scale is not None:
        if passages.dtype != torch.float16 or passages.shape[1] % 2:
            raise _lib.MatchmakerB200Error("flat_ip_topk: split storage is [n, 2*dim] fp16")
        dim = passages.shape[1] // 2
        if queries.shape[1] != dim:
            raise _lib.MatchmakerB200Error(f"flat_ip_topk: queries have dim {queries.shape[1]}, split passages {dim}")
        queries, sq = flat_ip_split_f32(queries, "queries")
        unscale = -(sq + split_scale)
        dcode = _lib.F32_SPLIT16
    else:
        if queries.shape[1] != passages.shape[1]:
            raise _lib.MatchmakerB200Error(f"flat_ip_topk: queries have dim {queries.shape[1]}, passages {passages.shape[1]}")
        queries = queries.to(passages.dtype).contiguous()
        dim = queries.shape[1]
        dcode = _lib.F8E4M3 if fp8 else _DTYPES[passages.dtype]
    passages = passages.contiguous()
    nq = queries.shape[0]
    if ids is not None:
        ids = ids.to(torch.int64).contiguous()
    if nq == 0 and 1 <= k <= FLAT_IP_MAX_K:   # as ivf_search: an empty batch has an empty result
        return (torch.empty((0, k), dtype=torch.float32, device=dev),
                torch.empty((0, k), dtype=torch.int64, device=dev))
    lib = _lib.load()
    with torch.cuda.device(dev):
        wsb = lib.mmb200_flat_ip_workspace_bytes(nq, n, k)
        if wsb <= 0:
            raise _lib.MatchmakerB200Error(f"flat_ip_topk: unsupported sizes nq={nq} n={n} k={k} (1 <= k <= {FLAT_IP_MAX_K}): "
                                           + _lib.last_error())
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        out_s = torch.empty((nq, k), dtype=torch.float32, device=dev)
        out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
        rc = lib.mmb200_flat_ip_topk(_ptr(queries), _ptr(passages), _ptr(ids), _ptr(out_s), _ptr(out_i), _ptr(ws), wsb,
                                     nq, n, dim, k, dcode, id_base, _stream(dev))
    _lib.check(rc, "mmb200_flat_ip_topk")
    if unscale is not None:
        # back to the unscaled domain: a power of two, exact; faiss's "no result" filler (-FLT_MAX) stays what it is
        out_s = torch.where(out_s > -3.0e38, torch.ldexp(out_s, torch.tensor(unscale, device=dev)), out_s)
    return out_s, out_i


def topk_merge(cand_scores: torch.Tensor, cand_ids: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per-query merge of candidate lists [nq, L] -> top-k under (score desc, id asc)."""
    dev = _require_cuda(cand_scores, cand_ids)
    cand_scores = cand_scores.to(torch.float32).contiguous()
    cand_ids = cand_ids.to(torch.int64).contiguous()
    nq, L = cand_scores.shape
    out_s = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_topk_merge(_ptr(cand_scores), _ptr(cand_ids), _ptr(out_s), _ptr(out_i), nq, L, k, _stream(dev))
    _lib.check(rc, "mmb200_topk_merge")
    return out_s, out_i


TOPK_UNIQUE_MAX_K = 4096


def topk_unique(cand_scores: torch.Tensor, cand_ids: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Per-query de-duplication + top-k of candidate lists [nq, L]: the k best DISTINCT ids, each with its highest
    score, under (score desc, id asc).  Void candidates (score NaN / -inf / -FLT_MAX) are dropped; missing results are
    (-FLT_MAX, -1).  1 <= k <= 4096."""
    dev = _require_cuda(cand_scores, cand_ids)
    cand_scores = cand_scores.to(torch.float32).contiguous()
    cand_ids = cand_ids.to(torch.int64).contiguous()
    nq, L = cand_scores.shape
    if tuple(cand_ids.shape) != (nq, L):
        raise _lib.MatchmakerB200Error(f"topk_unique: scores {tuple(cand_scores.shape)} vs ids {tuple(cand_ids.shape)}")
    out_s = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_topk_unique(_ptr(cand_scores), _ptr(cand_ids), _ptr(out_s), _ptr(out_i), nq, L, k, _stream(dev))
    _lib.check(rc, "mmb200_topk_unique")
    return out_s, out_i


IVF_MAX_PROBE = 1024
# Device scratch one ivf_search call may take.  The scratch grows with nq * nprobe (gathered queries, one candidate slot
# per (query, probe)), so larger query sets are searched in batches that fit.
IVF_WORKSPACE_CAP = 2 << 30


def ivf_query_batch(nq: int, workspace_bytes, cap: int) -> int:
    """Queries per ivf_search batch: nq halved until `workspace_bytes(batch)` fits `cap` (at least one query).  A size of
    0 means the batch is outside the envelope (nq * nprobe too large), so it is halved as well."""
    b = max(1, nq)
    while b > 1 and not 0 < workspace_bytes(b) <= cap:
        b = (b + 1) // 2
    return b


def ivf_search(queries: torch.Tensor, rows: torch.Tensor, ids: torch.Tensor, list_offsets: torch.Tensor,
               probes: torch.Tensor, k: int, max_list_len: int, split_scale: Optional[int] = None,
               row_index: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exact inner-product top-k over the union of each query's probed lists (faiss IndexIVF search semantics).

    rows [n, dim] fp16 / bf16, sorted by list: list l is rows ``list_offsets[l]:list_offsets[l+1]`` (int64 [nlist+1]);
    ids [n] int64 user ids; probes [nq, nprobe] int64 list ids, distinct per row (ids outside [0, nlist) probe nothing);
    max_list_len bounds every list's length.  Returns (scores [nq, k] f32, ids [nq, k] int64) under (score desc, id asc),
    with a (-3.4028235e38, -1) tail when the probed lists hold fewer than k rows.  fp32 storage: ``rows`` =
    flat_ip_split_f32(x, "passages")[0] with its scale as ``split_scale``, as for flat_ip_topk.  1 <= k <= 1024,
    1 <= nprobe <= 1024.  Queries are searched in batches whose scratch fits IVF_WORKSPACE_CAP.

    row_index (int64 [list_offsets[-1]], optional): the rows are NOT sorted by list; list position p is row
    ``row_index[p]`` of ``rows``, and ``ids`` is indexed by row (mmb200_ivf_search_gather).  The result equals the call
    without row_index over ``rows[row_index]`` with ids ``ids[row_index]``, without that copy of the rows.

    E4M3 (queries and rows torch.float8_e4m3fn, with row_index only): scores in the scaled domain, as flat_ip_topk."""
    dev = _require_cuda(queries, rows, ids, list_offsets, probes, row_index)
    fp8 = _fp8_pair(queries, rows, "ivf_search")
    if fp8 and row_index is None:
        raise _lib.MatchmakerB200Error("ivf_search: e4m3 rows are scanned in place through row_index only")
    if not fp8 and rows.dtype not in (torch.float16, torch.bfloat16):
        raise _lib.MatchmakerB200Error("ivf_search: rows must be fp16 / bf16, or the fp16 split of fp32 (flat_ip_split_f32)")
    if probes.dim() != 2 or probes.shape[0] != queries.shape[0]:
        raise _lib.MatchmakerB200Error(f"ivf_search: probes must be [nq, nprobe], got {tuple(probes.shape)}")
    nq, nprobe = probes.shape
    nlist = list_offsets.numel() - 1
    unscale = None
    if split_scale is not None:
        if rows.dtype != torch.float16 or rows.shape[1] % 2:
            raise _lib.MatchmakerB200Error("ivf_search: split storage is [n, 2*dim] fp16")
        dim = rows.shape[1] // 2
        if queries.shape[1] != dim:
            raise _lib.MatchmakerB200Error(f"ivf_search: queries have dim {queries.shape[1]}, split rows {dim}")
        queries, sq = flat_ip_split_f32(queries, "queries")
        unscale = -(sq + split_scale)
        dcode = _lib.F32_SPLIT16
    else:
        if queries.shape[1] != rows.shape[1]:
            raise _lib.MatchmakerB200Error(f"ivf_search: queries have dim {queries.shape[1]}, rows {rows.shape[1]}")
        queries = queries.to(rows.dtype).contiguous()
        dim = queries.shape[1]
        dcode = _lib.F8E4M3 if fp8 else _DTYPES[rows.dtype]
    if ids.numel() != rows.shape[0] or list_offsets.dim() != 1 or nlist < 1:
        raise _lib.MatchmakerB200Error(f"ivf_search: {ids.numel()} ids for {rows.shape[0]} rows, list_offsets "
                                       f"{tuple(list_offsets.shape)} (need [nlist + 1], nlist >= 1)")
    if row_index is not None:
        if row_index.dim() != 1 or row_index.numel() > rows.shape[0]:
            raise _lib.MatchmakerB200Error(f"ivf_search: row_index must be [list_offsets[-1]] (at most one entry per row), "
                                           f"got {tuple(row_index.shape)} for {rows.shape[0]} rows")
        row_index = row_index.to(torch.int64).contiguous()
    rows, probes = rows.contiguous(), probes.to(torch.int64).contiguous()
    ids, list_offsets = ids.to(torch.int64).contiguous(), list_offsets.to(torch.int64).contiguous()
    out_s = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
    if nq == 0:
        return out_s, out_i
    lib = _lib.load()
    with torch.cuda.device(dev):
        def wsb(b):
            return lib.mmb200_ivf_workspace_bytes(b, nprobe, nlist, max_list_len, dim, k, dcode)
        if wsb(1) <= 0:
            raise _lib.MatchmakerB200Error(f"ivf_search: unsupported sizes nprobe={nprobe} nlist={nlist} dim={dim} k={k} "
                                           f"(1 <= k <= {FLAT_IP_MAX_K}, 1 <= nprobe <= {IVF_MAX_PROBE}, dim % 64 == 0; "
                                           "e4m3: dim % 128 == 0, 128 <= dim <= 1024)")
        b = ivf_query_batch(nq, wsb, IVF_WORKSPACE_CAP)
        ws = torch.empty(wsb(b), dtype=torch.uint8, device=dev)
        for b0 in range(0, nq, b):
            b1 = min(nq, b0 + b)
            tail = (_ptr(probes[b0:b1]), _ptr(out_s[b0:b1]), _ptr(out_i[b0:b1]), _ptr(ws), ws.numel(), b1 - b0, nprobe,
                    nlist, rows.shape[0], max_list_len, dim, k, dcode, _stream(dev))
            if row_index is None:
                rc = lib.mmb200_ivf_search(_ptr(queries[b0:b1]), _ptr(rows), _ptr(ids), _ptr(list_offsets), *tail)
                _lib.check(rc, "mmb200_ivf_search")
            else:
                rc = lib.mmb200_ivf_search_gather(_ptr(queries[b0:b1]), _ptr(rows), _ptr(ids), _ptr(row_index),
                                                  _ptr(list_offsets), *tail)
                _lib.check(rc, "mmb200_ivf_search_gather")
    if unscale is not None:
        out_s = torch.where(out_s > -3.0e38, torch.ldexp(out_s, torch.tensor(unscale, device=dev)), out_s)
    return out_s, out_i


def ivf_list_means(x: torch.Tensor, perm: torch.Tensor, offsets: torch.Tensor) -> torch.Tensor:
    """Spherical k-means update: row l = normalised mean of x[perm[offsets[l]:offsets[l+1]]] ([nlist, dim] f32), summed
    in that order in fp64, so it is bit-reproducible; an empty list gives a zero row.  x [n, dim] fp16 / bf16 / fp32."""
    dev = _require_cuda(x, perm, offsets)
    if x.dtype not in _DTYPES:
        raise _lib.MatchmakerB200Error(f"ivf_list_means: x must be fp16 / bf16 / fp32, got {x.dtype}")
    x, perm, offsets = x.contiguous(), perm.to(torch.int64).contiguous(), offsets.to(torch.int64).contiguous()
    nlist = offsets.numel() - 1
    out = torch.empty((nlist, x.shape[1]), dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_ivf_list_means(_ptr(x), _ptr(perm), _ptr(offsets), _ptr(out), nlist, x.shape[1], _DTYPES[x.dtype],
                                       _stream(dev))
    _lib.check(rc, "mmb200_ivf_list_means")
    return out


RESIDUAL_BITS = (1, 2)


def _residual_tables(base: torch.Tensor, weight: torch.Tensor, bits: int, dim: int, what: str):
    if bits not in RESIDUAL_BITS:
        raise _lib.MatchmakerB200Error(f"{what}: bits must be 1 or 2, got {bits}")
    if dim % 64 or not 64 <= dim <= 1024:
        raise _lib.MatchmakerB200Error(f"{what}: residual codes need dim % 64 == 0 and 64 <= dim <= 1024, got {dim}")
    if base.dtype != torch.float16 or base.dim() != 2 or base.shape[1] != dim:
        raise _lib.MatchmakerB200Error(f"{what}: base must be [nlist, {dim}] fp16, got {tuple(base.shape)} {base.dtype}")
    if weight is not None and (weight.dtype != torch.float16 or tuple(weight.shape) != (dim, 1 << bits)):
        raise _lib.MatchmakerB200Error(f"{what}: weight must be [{dim}, {1 << bits}] fp16, got {tuple(weight.shape)} "
                                       f"{weight.dtype}")
    return base.contiguous(), None if weight is None else weight.contiguous()


def _residual_codes(codes: torch.Tensor, dim: int, bits: int, what: str) -> torch.Tensor:
    if codes.dtype != torch.uint8 or codes.dim() != 2 or codes.shape[1] != dim * bits // 8:
        raise _lib.MatchmakerB200Error(f"{what}: codes must be [n_rows, {dim * bits // 8}] uint8, got "
                                       f"{tuple(codes.shape)} {codes.dtype}")
    return codes.contiguous()


def _residual_list_ids(list_ids: torch.Tensor, n_rows: int, nlist: int, what: str) -> torch.Tensor:
    if list_ids.dim() != 1 or list_ids.numel() != n_rows:
        raise _lib.MatchmakerB200Error(f"{what}: list_ids must be [{n_rows}], got {tuple(list_ids.shape)}")
    list_ids = list_ids.to(torch.int32).contiguous()
    if n_rows and not (0 <= int(list_ids.min()) and int(list_ids.max()) < nlist):
        raise _lib.MatchmakerB200Error(f"{what}: list ids must lie in [0, {nlist})")
    return list_ids


def residual_encode(rows: torch.Tensor, list_ids: torch.Tensor, base: torch.Tensor, cutoff: torch.Tensor,
                    bits: int) -> torch.Tensor:
    """Residual codes [n, dim * bits / 8] uint8 of fp16 rows [n, dim] of lists ``list_ids`` (int [n], in [0, nlist)):
    code[d] = #{i : cutoff[d][i] <= float(x[d]) - float(base[l][d])} in fp32, ``bits`` (1 or 2) bits per dimension,
    dimension d in bits [bits * (d % (8 / bits)), +bits) of byte d * bits / 8.  base [nlist, dim] fp16, cutoff
    [dim, 2^bits - 1] fp32 ascending.  dim % 64 == 0, 64 <= dim <= 1024."""
    dev = _require_cuda(rows, list_ids, base, cutoff)
    if rows.dtype != torch.float16 or rows.dim() != 2:
        raise _lib.MatchmakerB200Error(f"residual_encode: rows must be [n, dim] fp16, got {tuple(rows.shape)} {rows.dtype}")
    n, dim = rows.shape
    base, _ = _residual_tables(base, None, bits, dim, "residual_encode")
    if cutoff.dtype != torch.float32 or tuple(cutoff.shape) != (dim, (1 << bits) - 1):
        raise _lib.MatchmakerB200Error(f"residual_encode: cutoff must be [{dim}, {(1 << bits) - 1}] fp32")
    list_ids = _residual_list_ids(list_ids, n, base.shape[0], "residual_encode")
    rows, cutoff = rows.contiguous(), cutoff.contiguous()
    out = torch.empty((n, dim * bits // 8), dtype=torch.uint8, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_residual_encode(_ptr(rows), _ptr(list_ids), _ptr(base), _ptr(cutoff), _ptr(out), n, dim, bits,
                                        _stream(dev))
    _lib.check(rc, "mmb200_residual_encode")
    return out


def residual_decode(codes: torch.Tensor, list_ids: torch.Tensor, base: torch.Tensor, weight: torch.Tensor,
                    bits: int) -> torch.Tensor:
    """fp16 rows [n, dim] of residual codes (:func:`residual_encode`): value[d] = fp16_rn(float(base[l][d]) +
    float(weight[d][code[d]])), weight [dim, 2^bits] fp16."""
    dev = _require_cuda(codes, list_ids, base, weight)
    dim = base.shape[1] if base.dim() == 2 else -1
    base, weight = _residual_tables(base, weight, bits, dim, "residual_decode")
    codes = _residual_codes(codes, dim, bits, "residual_decode")
    n = codes.shape[0]
    list_ids = _residual_list_ids(list_ids, n, base.shape[0], "residual_decode")
    out = torch.empty((n, dim), dtype=torch.float16, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_residual_decode(_ptr(codes), _ptr(list_ids), _ptr(base), _ptr(weight), _ptr(out), n, dim, bits,
                                        _stream(dev))
    _lib.check(rc, "mmb200_residual_decode")
    return out


def ivf_search_residual(queries: torch.Tensor, codes: torch.Tensor, base: torch.Tensor, weight: torch.Tensor,
                        bits: int, ids: torch.Tensor, row_index: torch.Tensor, list_offsets: torch.Tensor,
                        probes: torch.Tensor, k: int, max_list_len: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """:func:`ivf_search` with ``row_index`` over residual codes instead of fp16 rows: list position p is code row
    ``row_index[p]``, which must belong to the list whose positions hold p.  Bit-identical to
    ``ivf_search(queries, residual_decode(codes, ...), ids, list_offsets, probes, k, max_list_len, row_index=row_index)``
    without materialising the decoded rows.  queries [nq, dim] (cast to fp16)."""
    dev = _require_cuda(queries, codes, base, weight, ids, row_index, list_offsets, probes)
    dim = base.shape[1] if base.dim() == 2 else -1
    base, weight = _residual_tables(base, weight, bits, dim, "ivf_search_residual")
    codes = _residual_codes(codes, dim, bits, "ivf_search_residual")
    nlist = list_offsets.numel() - 1
    if queries.dim() != 2 or queries.shape[1] != dim:
        raise _lib.MatchmakerB200Error(f"ivf_search_residual: queries must be [nq, {dim}], got {tuple(queries.shape)}")
    if probes.dim() != 2 or probes.shape[0] != queries.shape[0]:
        raise _lib.MatchmakerB200Error(f"ivf_search_residual: probes must be [nq, nprobe], got {tuple(probes.shape)}")
    if ids.numel() != codes.shape[0] or list_offsets.dim() != 1 or nlist != base.shape[0]:
        raise _lib.MatchmakerB200Error(f"ivf_search_residual: {ids.numel()} ids for {codes.shape[0]} rows, "
                                       f"list_offsets {tuple(list_offsets.shape)} for {base.shape[0]} bases")
    if row_index.dim() != 1 or row_index.numel() > codes.shape[0]:
        raise _lib.MatchmakerB200Error(f"ivf_search_residual: row_index must be [list_offsets[-1]], got "
                                       f"{tuple(row_index.shape)} for {codes.shape[0]} rows")
    nq, nprobe = probes.shape
    queries = queries.to(torch.float16).contiguous()
    probes, ids = probes.to(torch.int64).contiguous(), ids.to(torch.int64).contiguous()
    row_index, list_offsets = row_index.to(torch.int64).contiguous(), list_offsets.to(torch.int64).contiguous()
    out_s = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
    if nq == 0:
        return out_s, out_i
    lib = _lib.load()
    with torch.cuda.device(dev):
        def wsb(b):
            return lib.mmb200_ivf_workspace_bytes(b, nprobe, nlist, max_list_len, dim, k, _lib.F16)
        if wsb(1) <= 0:
            raise _lib.MatchmakerB200Error(f"ivf_search_residual: unsupported sizes nprobe={nprobe} nlist={nlist} k={k} "
                                           f"(1 <= k <= {FLAT_IP_MAX_K}, 1 <= nprobe <= {IVF_MAX_PROBE})")
        b = ivf_query_batch(nq, wsb, IVF_WORKSPACE_CAP)
        ws = torch.empty(wsb(b), dtype=torch.uint8, device=dev)
        for b0 in range(0, nq, b):
            b1 = min(nq, b0 + b)
            rc = lib.mmb200_ivf_search_residual(_ptr(queries[b0:b1]), _ptr(codes), _ptr(base), _ptr(weight), bits,
                                                _ptr(ids), _ptr(row_index), _ptr(list_offsets), _ptr(probes[b0:b1]),
                                                _ptr(out_s[b0:b1]), _ptr(out_i[b0:b1]), _ptr(ws), ws.numel(), b1 - b0,
                                                nprobe, nlist, codes.shape[0], max_list_len, dim, k, _stream(dev))
            _lib.check(rc, "mmb200_ivf_search_residual")
    return out_s, out_i


def maxsim_store_residual(q: torch.Tensor, codes: torch.Tensor, list_ids: torch.Tensor, base: torch.Tensor,
                          weight: torch.Tensor, bits: int, doc_offsets: torch.Tensor, pair_q: torch.Tensor,
                          pair_d: torch.Tensor, max_doc_len: int) -> torch.Tensor:
    """:func:`maxsim_store` over residual codes (row r of list ``list_ids[r]``), fp32 [n_pairs]: bit-identical to
    ``maxsim_store(q, residual_decode(codes, ...), doc_offsets, pair_q, pair_d, max_doc_len, impl="tcgen05_docm")``.
    q [n_q, Lq, dim] (cast to fp16), 1 <= Lq <= 128."""
    dev = _require_cuda(q, codes, list_ids, base, weight, doc_offsets, pair_q, pair_d)
    dim = base.shape[1] if base.dim() == 2 else -1
    base, weight = _residual_tables(base, weight, bits, dim, "maxsim_store_residual")
    codes = _residual_codes(codes, dim, bits, "maxsim_store_residual")
    if q.dim() != 3 or q.shape[-1] != dim:
        raise _lib.MatchmakerB200Error(f"maxsim_store_residual: q must be [n_q, Lq, {dim}], got {tuple(q.shape)}")
    if list_ids.dim() != 1 or list_ids.numel() != codes.shape[0]:
        raise _lib.MatchmakerB200Error("maxsim_store_residual: one list id per code row")
    q = q.to(torch.float16).contiguous()
    list_ids = list_ids.to(torch.int32).contiguous()
    doc_offsets = doc_offsets.to(torch.int64).contiguous()
    pair_q = pair_q.to(torch.int32).contiguous().view(-1)
    pair_d = pair_d.to(torch.int32).contiguous().view(-1)
    if pair_q.numel() != pair_d.numel():
        raise _lib.MatchmakerB200Error("pair_q / pair_d length mismatch")
    n_q, Lq, _ = q.shape
    out = torch.empty(pair_q.numel(), dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_maxsim_store_residual_fwd(_ptr(q), _ptr(codes), _ptr(list_ids), _ptr(base), _ptr(weight), bits,
                                                  _ptr(doc_offsets), _ptr(pair_q), _ptr(pair_d), _ptr(out), n_q,
                                                  codes.shape[0], doc_offsets.numel() - 1, pair_q.numel(), Lq,
                                                  int(max_doc_len), dim, _stream(dev))
    _lib.check(rc, "mmb200_maxsim_store_residual_fwd")
    return out


PLAID_MAX_LQ = 128
PLAID_MAX_NLIST = 1 << 18
PLAID_MAX_QUERIES = 65535   # queries per launch (grid y)


def plaid_lqp(lq: int) -> int:
    """Width of a query's centroid score row: Lq rounded up to a multiple of 32."""
    return 32 * ((lq + 31) // 32)


def _plaid_envelope(lq: int, nlist: int, what: str, dim: Optional[int] = None):
    if not 1 <= lq <= PLAID_MAX_LQ:
        raise _lib.MatchmakerB200Error(f"{what}: PLAID needs 1 <= Lq <= {PLAID_MAX_LQ}, got {lq}")
    if not 1 <= nlist <= PLAID_MAX_NLIST:
        raise _lib.MatchmakerB200Error(f"{what}: PLAID needs 1 <= nlist <= 2^18, got {nlist}")
    if dim is not None and (dim % 64 or not 64 <= dim <= 1024):
        raise _lib.MatchmakerB200Error(f"{what}: PLAID needs dim % 64 == 0 and 64 <= dim <= 1024, got {dim}")


def plaid_centroid_scores(q: torch.Tensor, centroids: torch.Tensor, threshold: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """PLAID's query x centroid table of queries q [nq, Lq, dim] and centroids [nlist, dim] (both cast to fp16):
    (scores [nq, nlist, LQP] fp16, scores[q][c][i] = fp16_rn(fp32 sum_d q[i][d] * centroid[c][d]), 0 for i >= Lq;
    keep [nq, ceil(nlist / 32)] int32 bitmask, bit c set when the max over the query's live tokens (rows with a nonzero
    fp16 element) of scores[q][c] is >= threshold).  threshold -inf keeps every centroid of a query with a live token.
    1 <= Lq <= 128, 1 <= nlist <= 2^18, dim % 64 == 0, 64 <= dim <= 1024."""
    dev = _require_cuda(q, centroids)
    if q.dim() != 3 or centroids.dim() != 2 or centroids.shape[1] != q.shape[2]:
        raise _lib.MatchmakerB200Error(f"plaid_centroid_scores: q [nq, Lq, dim] and centroids [nlist, dim], got "
                                       f"{tuple(q.shape)} and {tuple(centroids.shape)}")
    nq, lq, dim = q.shape
    nlist = centroids.shape[0]
    _plaid_envelope(lq, nlist, "plaid_centroid_scores", dim)
    if threshold != threshold:
        raise _lib.MatchmakerB200Error("plaid_centroid_scores: the centroid score threshold is NaN")
    q, centroids = q.to(torch.float16).contiguous(), centroids.to(torch.float16).contiguous()
    scores = torch.empty((nq, nlist, plaid_lqp(lq)), dtype=torch.float16, device=dev)
    keep = torch.empty((nq, (nlist + 31) // 32), dtype=torch.int32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        for b0 in range(0, nq, PLAID_MAX_QUERIES):
            b1 = min(nq, b0 + PLAID_MAX_QUERIES)
            rc = lib.mmb200_plaid_centroid_scores(_ptr(q[b0:b1]), _ptr(centroids), _ptr(scores[b0:b1]), _ptr(keep[b0:b1]),
                                                  b1 - b0, lq, nlist, dim, float(threshold), _stream(dev))
            _lib.check(rc, "mmb200_plaid_centroid_scores")
    return scores, keep


def plaid_candidates(probes: torch.Tensor, plist_offsets: torch.Tensor, plist_pids: torch.Tensor, n_docs: int, cap: int,
                     first_doc: int = 0) -> torch.Tensor:
    """The candidate passages of every query: probes [nq, n_probes] int64 list ids (entries outside [0, nlist) probe
    nothing); list l holds local passages plist_pids[plist_offsets[l]:plist_offsets[l+1]] (int32 in [0, n_docs)).
    Returns [nq, cap] int64: the union of the probed lists' passages as first_doc + pid, ascending, then -1.  A union
    larger than cap keeps its cap smallest ids: cap = min(n_docs, n_probes * longest list) never truncates."""
    dev = _require_cuda(probes, plist_offsets, plist_pids)
    if probes.dim() != 2 or plist_offsets.dim() != 1 or plist_offsets.numel() < 2 or plist_pids.dim() != 1:
        raise _lib.MatchmakerB200Error("plaid_candidates: probes [nq, n_probes], plist_offsets [nlist + 1], plist_pids [n]")
    if not 1 <= cap <= max(n_docs, 1):
        raise _lib.MatchmakerB200Error(f"plaid_candidates: cap must be in [1, max(n_docs, 1)], got {cap}")
    nq, n_probes = probes.shape
    probes, plist_offsets = probes.to(torch.int64).contiguous(), plist_offsets.to(torch.int64).contiguous()
    plist_pids = plist_pids.to(torch.int32).contiguous()
    out = torch.empty((nq, cap), dtype=torch.int64, device=dev)
    if nq == 0 or n_probes == 0:
        return out.fill_(-1)
    bitmap = torch.empty(nq * max(1, (n_docs + 31) // 32), dtype=torch.int32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_plaid_candidates(_ptr(probes), _ptr(plist_offsets), _ptr(plist_pids), _ptr(bitmap), _ptr(out), nq,
                                         n_probes, plist_offsets.numel() - 1, n_docs, cap, first_doc, _stream(dev))
    _lib.check(rc, "mmb200_plaid_candidates")
    return out


def plaid_interaction(scores: torch.Tensor, keep: Optional[torch.Tensor], list_ids: torch.Tensor,
                      doc_offsets: torch.Tensor, cand: torch.Tensor, lq: int, first_doc: int = 0) -> torch.Tensor:
    """Centroid interaction [nq, C] f32 of candidates cand [nq, C] (global ids; ids outside [first_doc, first_doc +
    n_docs) are void): the sum over query tokens i < lq of the max over the passage's rows r of
    float(scores[q][list_ids[r]][i]), over the rows whose list is kept in ``keep`` (pruned; None: every row); -inf
    when no row qualifies or the candidate is void.  scores, keep: :func:`plaid_centroid_scores`; list_ids [n_rows]
    int32; doc_offsets [n_docs + 1] int64.  Bit-reproducible (fixed-order sums)."""
    dev = _require_cuda(scores, keep, list_ids, doc_offsets, cand)
    if scores.dim() != 3 or scores.dtype != torch.float16 or cand.dim() != 2 or cand.shape[0] != scores.shape[0]:
        raise _lib.MatchmakerB200Error(f"plaid_interaction: scores [nq, nlist, LQP] fp16 and cand [nq, C], got "
                                       f"{tuple(scores.shape)} {scores.dtype} and {tuple(cand.shape)}")
    nq, nlist, lqp = scores.shape
    _plaid_envelope(lq, nlist, "plaid_interaction")
    if lqp != plaid_lqp(lq):
        raise _lib.MatchmakerB200Error(f"plaid_interaction: score rows of {lqp} for Lq {lq} (need {plaid_lqp(lq)})")
    if keep is not None and tuple(keep.shape) != (nq, (nlist + 31) // 32):
        raise _lib.MatchmakerB200Error(f"plaid_interaction: keep must be [{nq}, {(nlist + 31) // 32}], got "
                                       f"{tuple(keep.shape)}")
    n_docs = doc_offsets.numel() - 1
    if list_ids.dim() != 1 or doc_offsets.dim() != 1 or n_docs < 0:
        raise _lib.MatchmakerB200Error("plaid_interaction: list_ids [n_rows], doc_offsets [n_docs + 1]")
    scores, cand = scores.contiguous(), cand.to(torch.int64).contiguous()
    list_ids, doc_offsets = list_ids.to(torch.int32).contiguous(), doc_offsets.to(torch.int64).contiguous()
    keep = None if keep is None else keep.contiguous()
    n_cand = cand.shape[1]
    out = torch.empty((nq, n_cand), dtype=torch.float32, device=dev)
    if nq == 0 or n_cand == 0:
        return out
    lib = _lib.load()
    with torch.cuda.device(dev):
        for b0 in range(0, nq, PLAID_MAX_QUERIES):
            b1 = min(nq, b0 + PLAID_MAX_QUERIES)
            rc = lib.mmb200_plaid_interaction(_ptr(scores[b0:b1]), None if keep is None else _ptr(keep[b0:b1]),
                                              _ptr(list_ids), _ptr(doc_offsets), _ptr(cand[b0:b1]), _ptr(out[b0:b1]),
                                              b1 - b0, lq, nlist, n_docs, n_cand, first_doc, int(keep is not None),
                                              _stream(dev))
            _lib.check(rc, "mmb200_plaid_interaction")
    return out


AH_MAX_KR = 1024
# Device scratch one ah_search call may take; it grows with nq * nprobe (one candidate slot per (query, probe)), so
# larger query sets are searched in batches that fit.
AH_WORKSPACE_CAP = 2 << 30


def ah_search(luts: torch.Tensor, codes: torch.Tensor, list_offsets: torch.Tensor, probes: torch.Tensor,
              bias: torch.Tensor, kr: int, max_list_len: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Approximate top-kr over each query's probed leaves from 4-bit AH codes (mmb200_ah_search).

    luts [nq, dim/2, 16] f32 lookup tables; codes [n, dim/4] uint8 sorted by leaf (leaf l is rows
    ``list_offsets[l]:list_offsets[l+1]``, block 2j in the low nibble of byte j, block 2j+1 in the high one); probes
    [nq, nprobe] int64 leaf ids (ids outside [0, nlist) probe nothing); bias [nq, nprobe] f32, each probed leaf's
    <query, centroid>.  Score = bias + sum over blocks ascending of luts[q, m, code], fp32.  Returns (approximate scores
    [nq, kr] f32, row positions [nq, kr] int64) under (score desc, position asc) with a (-3.4028235e38, -1) tail.
    1 <= kr <= 1024, 1 <= nprobe <= 1024, dim % 64 == 0.  Queries are searched in batches whose scratch fits
    AH_WORKSPACE_CAP.  No host synchronisation."""
    dev = _require_cuda(luts, codes, list_offsets, probes, bias)
    if codes.dtype != torch.uint8 or codes.dim() != 2:
        raise _lib.MatchmakerB200Error("ah_search: codes must be [n, dim/4] uint8")
    n, dim = codes.shape[0], codes.shape[1] * 4
    if probes.dim() != 2 or luts.shape != (probes.shape[0], dim // 2, 16) or bias.shape != probes.shape:
        raise _lib.MatchmakerB200Error(f"ah_search: luts {tuple(luts.shape)}, probes {tuple(probes.shape)} and bias "
                                       f"{tuple(bias.shape)} do not fit codes for dim {dim}")
    nq, nprobe = probes.shape
    nlist = list_offsets.numel() - 1
    luts, codes = luts.to(torch.float32).contiguous(), codes.contiguous()
    probes, bias = probes.to(torch.int64).contiguous(), bias.to(torch.float32).contiguous()
    list_offsets = list_offsets.to(torch.int64).contiguous()
    out_s = torch.empty((nq, kr), dtype=torch.float32, device=dev)
    out_p = torch.empty((nq, kr), dtype=torch.int64, device=dev)
    if nq == 0:
        return out_s, out_p
    lib = _lib.load()
    with torch.cuda.device(dev):
        def wsb(b):
            return lib.mmb200_ah_workspace_bytes(b, nprobe, nlist, max_list_len, dim, kr)
        if wsb(1) <= 0:
            raise _lib.MatchmakerB200Error(f"ah_search: unsupported sizes nprobe={nprobe} nlist={nlist} dim={dim} kr={kr} "
                                           f"(1 <= kr <= {AH_MAX_KR}, 1 <= nprobe <= {IVF_MAX_PROBE}, dim % 64 == 0)")
        b = ivf_query_batch(nq, wsb, AH_WORKSPACE_CAP)
        ws = torch.empty(wsb(b), dtype=torch.uint8, device=dev)
        for b0 in range(0, nq, b):
            b1 = min(nq, b0 + b)
            rc = lib.mmb200_ah_search(_ptr(luts[b0:b1]), _ptr(codes), _ptr(list_offsets), _ptr(probes[b0:b1]),
                                      _ptr(bias[b0:b1]), _ptr(out_s[b0:b1]), _ptr(out_p[b0:b1]), _ptr(ws), ws.numel(),
                                      b1 - b0, nprobe, nlist, n, max_list_len, dim, kr, _stream(dev))
            _lib.check(rc, "mmb200_ah_search")
    return out_s, out_p


def ah_reorder(queries: torch.Tensor, rows: torch.Tensor, ids: Optional[torch.Tensor], shortlist: torch.Tensor,
               top_n: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Exact re-scoring of a shortlist (mmb200_ah_reorder): rows [n, dim] fp16 or fp32 (queries are cast to it),
    shortlist [nq, kr] int64 row positions (-1 = void), ids [n] int64 user ids.  Every score is one fixed-order fp32
    formula.  Returns (scores [nq, top_n] f32, ids [nq, top_n] int64) under (score desc, id asc) with a
    (-3.4028235e38, -1) tail.  1 <= top_n <= kr <= 1024.  No host synchronisation."""
    dev = _require_cuda(queries, rows, ids, shortlist)
    if rows.dtype not in (torch.float16, torch.float32) or rows.dim() != 2:
        raise _lib.MatchmakerB200Error("ah_reorder: rows must be [n, dim] fp16 or fp32")
    n, dim = rows.shape
    if queries.dim() != 2 or queries.shape[1] != dim or shortlist.dim() != 2 or shortlist.shape[0] != queries.shape[0]:
        raise _lib.MatchmakerB200Error(f"ah_reorder: queries {tuple(queries.shape)}, shortlist {tuple(shortlist.shape)} "
                                       f"for rows of dim {dim}")
    nq, kr = shortlist.shape
    if not 1 <= top_n <= kr <= AH_MAX_KR:
        raise _lib.MatchmakerB200Error(f"ah_reorder: need 1 <= top_n <= kr <= {AH_MAX_KR}, got top_n={top_n} kr={kr}")
    queries, rows = queries.to(rows.dtype).contiguous(), rows.contiguous()
    shortlist = shortlist.to(torch.int64).contiguous()
    if ids is not None:
        ids = ids.to(torch.int64).contiguous()
    out_s = torch.empty((nq, top_n), dtype=torch.float32, device=dev)
    out_i = torch.empty((nq, top_n), dtype=torch.int64, device=dev)
    if nq == 0:
        return out_s, out_i
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_ah_reorder(_ptr(queries), _ptr(rows), _ptr(ids), _ptr(shortlist), _ptr(out_s), _ptr(out_i), nq, n,
                                   dim, kr, int(top_n), _DTYPES[rows.dtype], _stream(dev))
    _lib.check(rc, "mmb200_ah_reorder")
    return out_s, out_i


GRAPH_MAX_DEGREE = 1024   # R, edges per node
GRAPH_MAX_KNN = 1023      # K, k-NN degree before pruning
GRAPH_MAX_LIST = 1024     # L, search list size


def graph_hash_slots(L: int, R: int) -> int:
    """Slots of the search kernel's visited hash for list size L and out-degree R (next_pow2(4 * (L + R)))."""
    return int(_lib.load().mmb200_graph_hash_slots(int(L), int(R)))


def graph_prune(knn: torch.Tensor, R: int) -> torch.Tensor:
    """Rank-based detour pruning of a k-NN graph: knn [n, K] int32 row positions in rank order (-1 = void) ->
    [n, R] int32, the R edges of each node with the fewest detours (ties by rank) in rank order, -1 padded.
    1 <= K <= 1023, 1 <= R <= 1024."""
    dev = _require_cuda(knn)
    if knn.dim() != 2:
        raise _lib.MatchmakerB200Error(f"graph_prune: knn must be [n, K], got {tuple(knn.shape)}")
    n, K = knn.shape
    if not (1 <= K <= GRAPH_MAX_KNN and 1 <= R <= GRAPH_MAX_DEGREE):
        raise _lib.MatchmakerB200Error(f"graph_prune: need 1 <= K <= {GRAPH_MAX_KNN} and 1 <= R <= {GRAPH_MAX_DEGREE}, "
                                       f"got K={K} R={R}")
    knn = knn.to(torch.int32).contiguous()
    out = torch.empty((n, R), dtype=torch.int32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_graph_prune(_ptr(knn), _ptr(out), n, K, int(R), _stream(dev))
    _lib.check(rc, "mmb200_graph_prune")
    return out


def graph_search(queries: torch.Tensor, rows: torch.Tensor, ids: torch.Tensor, graph: torch.Tensor,
                 entries: torch.Tensor, k: int, L: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Beam search over a graph index, one CTA per query.

    rows [n, dim] fp16 or fp32 (queries are cast to it); graph [n, R] int32 row positions (-1 = no edge); entries
    [nq, m] int64 row positions that seed each query's list (1 <= m <= L); ids [n] int64 user ids.  The list keeps the
    L best rows seen under (score desc, position asc), and every score comes from one fixed-order fp32 formula.
    Returns (scores [nq, k] f32, ids [nq, k] int64) with a (-3.4028235e38, -1) tail where fewer than k rows were
    reached.  32 <= L <= 1024 (a multiple of 32), 1 <= k <= L.  No host synchronisation."""
    dev = _require_cuda(queries, rows, ids, graph, entries)
    if rows.dtype not in (torch.float16, torch.float32) or rows.dim() != 2:
        raise _lib.MatchmakerB200Error("graph_search: rows must be [n, dim] fp16 or fp32")
    n, dim = rows.shape
    if queries.dim() != 2 or queries.shape[1] != dim:
        raise _lib.MatchmakerB200Error(f"graph_search: queries have shape {tuple(queries.shape)}, rows dim {dim}")
    nq = queries.shape[0]
    if graph.dim() != 2 or graph.shape[0] != n or ids.numel() != n:
        raise _lib.MatchmakerB200Error(f"graph_search: graph {tuple(graph.shape)} and {ids.numel()} ids for {n} rows")
    if entries.dim() != 2 or entries.shape[0] != nq:
        raise _lib.MatchmakerB200Error(f"graph_search: entries must be [nq, m], got {tuple(entries.shape)}")
    if not (32 <= L <= GRAPH_MAX_LIST and L % 32 == 0 and 1 <= k <= L and 1 <= entries.shape[1] <= L):
        raise _lib.MatchmakerB200Error(f"graph_search: need 32 <= L <= {GRAPH_MAX_LIST} (a multiple of 32), 1 <= k <= L "
                                       f"and 1 <= entries <= L, got L={L} k={k} entries={entries.shape[1]}")
    queries = queries.to(rows.dtype).contiguous()
    rows, graph = rows.contiguous(), graph.to(torch.int32).contiguous()
    ids, entries = ids.to(torch.int64).contiguous(), entries.to(torch.int64).contiguous()
    out_s = torch.empty((nq, k), dtype=torch.float32, device=dev)
    out_i = torch.empty((nq, k), dtype=torch.int64, device=dev)
    if nq == 0:
        return out_s, out_i
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_graph_search(_ptr(queries), _ptr(rows), _ptr(ids), _ptr(graph), _ptr(entries), _ptr(out_s),
                                     _ptr(out_i), nq, n, dim, graph.shape[1], entries.shape[1], int(L), int(k),
                                     _DTYPES[rows.dtype], _stream(dev))
    _lib.check(rc, "mmb200_graph_search")
    return out_s, out_i


def maxsim_store(q: torch.Tensor, store: torch.Tensor, doc_offsets: torch.Tensor, pair_q: torch.Tensor,
                 pair_d: torch.Tensor, max_doc_len: int, impl: str = "auto") -> torch.Tensor:
    """ColBERT max-sim against a ragged token store, fp32 [n_pairs] (colbert.py:100-112, no masks).

    store [n_rows, dim]; passage d is rows ``doc_offsets[d] : doc_offsets[d+1]`` (int64 [n_docs+1], non-decreasing,
    at most ``max_doc_len`` rows read).  Pair p scores query ``pair_q[p]`` of q [n_q, Lq, dim] against passage
    ``pair_d[p]``; ``pair_d[p] < 0`` and passages without rows score -inf.  Same kernels and bit-identical scores as
    :func:`maxsim` on the passages padded to ``max_doc_len`` with a mask.

    E4M3 (q and store torch.float8_e4m3fn, 1 <= Lq <= 128, dim % 128 == 0, 128 <= dim <= 1024; impl "auto" or
    "tcgen05_docm"): the documents-on-M tensor-core kernel, scores in the scaled domain of :func:`fp8_quantize`."""
    dev = _require_cuda(q, store, doc_offsets, pair_q, pair_d)
    fp8 = _fp8_pair(q, store, "maxsim_store")
    if not fp8 and (q.dtype != store.dtype or q.dtype not in _DTYPES):
        raise _lib.MatchmakerB200Error(f"q/store must share a dtype in fp16/bf16/fp32, got {q.dtype}, {store.dtype}")
    if q.dim() != 3 or store.dim() != 2 or q.shape[-1] != store.shape[-1]:
        raise _lib.MatchmakerB200Error(f"expected q [n_q,Lq,dim], store [n_rows,dim]; got {tuple(q.shape)}, "
                                       f"{tuple(store.shape)}")
    q, store = q.contiguous(), store.contiguous()
    doc_offsets = doc_offsets.to(torch.int64).contiguous()
    pair_q = pair_q.to(torch.int32).contiguous().view(-1)
    pair_d = pair_d.to(torch.int32).contiguous().view(-1)
    if pair_q.numel() != pair_d.numel():
        raise _lib.MatchmakerB200Error("pair_q / pair_d length mismatch")
    n_q, Lq, dim = q.shape
    out = torch.empty(pair_q.numel(), dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_maxsim_store_fwd(_ptr(q), _ptr(store), _ptr(doc_offsets), _ptr(pair_q), _ptr(pair_d), _ptr(out),
                                         n_q, store.shape[0], doc_offsets.numel() - 1, pair_q.numel(), Lq, int(max_doc_len),
                                         dim, _lib.F8E4M3 if fp8 else _DTYPES[q.dtype], _IMPLS[impl], _stream(dev))
    _lib.check(rc, "mmb200_maxsim_store_fwd")
    return out


def _tkl_slot_map(packed_indices: torch.Tensor) -> torch.Tensor:
    """Packed index of every chunk slot (-1 = dropped by the packing), one kernel launch (mmb200_tkl_slot_map)."""
    pk = packed_indices.reshape(-1)
    if pk.dtype not in (torch.bool, torch.uint8):
        pk = pk != 0
    pk = pk.contiguous()
    out = torch.empty(pk.numel(), dtype=torch.int32, device=pk.device)
    lib = _lib.load()
    with torch.cuda.device(pk.device):
        rc = lib.mmb200_tkl_slot_map(_ptr(pk), _ptr(out), pk.numel(), _stream(pk.device))
    _lib.check(rc, "mmb200_tkl_slot_map")
    return out


def tkl_bwd(q_ctx, q_mask, doc_chunks, chunk_mask, packed_indices, chunk_pieces, mu, sigma, dense_weight, saturation,
            sat_params, sat_red_weight, chunk_scoring, top_idx, orig_score, grad_score):
    """Gradients of the TKL interaction stage: returns (grad_q_ctx, grad_doc_chunks, grad_dense_weight [K],
    grad_chunk_scoring [15], grad_sat_params, grad_sat_red_weight or None).

    Envelope: 1 <= Lq <= 40, 1 <= K <= 16, D a multiple of 4 up to what the kernel's shared-memory plan holds, D <= 356
    on an H100 (227 KB per block); outside it the call raises MatchmakerB200Error before any launch.  The forward accepts
    wider D through the tensor-core kernel, so a model with D > 356 can score but not train."""
    dev = _require_cuda(q_ctx, doc_chunks, grad_score)
    q_ctx = q_ctx.float().contiguous()
    doc_chunks = doc_chunks.float().contiguous()
    B, Lq, D = q_ctx.shape
    C = int(chunk_pieces)
    slot = _tkl_slot_map(packed_indices)
    q_mask, chunk_mask, mcode = _common_mask_dtype(_prep_mask(q_mask), _prep_mask(chunk_mask))
    mu, sigma, dense_weight = _f32c(mu).view(-1), _f32c(sigma).view(-1), _f32c(dense_weight).view(-1)
    sat_params = _f32c(sat_params).view(-1)
    red = None if sat_red_weight is None else _f32c(sat_red_weight).view(-1)
    K = mu.numel()
    sat_code = {"embedding": 0, "log": 1}[saturation]
    n_sat = 13 if sat_code == 0 else K
    stride = K + 15 + n_sat + (D if sat_code == 0 else 0)
    gq = torch.empty_like(q_ctx)
    gc = torch.empty_like(doc_chunks)
    gp = torch.empty(stride, dtype=torch.float32, device=dev)
    ws = torch.empty(max(1, B) * stride, dtype=torch.float32, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        rc = lib.mmb200_tkl_bwd(_ptr(q_ctx), _ptr(q_mask), _ptr(doc_chunks), _ptr(chunk_mask), _ptr(slot), _ptr(mu),
                                _ptr(sigma), _ptr(dense_weight), _ptr(red), _ptr(sat_params),
                                _ptr(_f32c(chunk_scoring).view(-1)), _ptr(top_idx.contiguous()),
                                _ptr(orig_score.contiguous()), _ptr(_f32c(grad_score)), _ptr(gq), _ptr(gc), _ptr(gp),
                                _ptr(ws), B, doc_chunks.shape[0], Lq, D, C, K, sat_code, mcode, _stream(dev))
    _lib.check(rc, "mmb200_tkl_bwd")
    g_dense, g_cs, g_sat = gp[:K], gp[K:K + 15], gp[K + 15:K + 15 + n_sat]
    g_red = gp[K + 15 + n_sat:] if sat_code == 0 else None
    return gq, gc, g_dense, g_cs, g_sat, g_red
