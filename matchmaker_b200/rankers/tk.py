"""TK (ECAI'20): transformer contextualisation in PyTorch + cosine / kernel pooling on the GPU kernel.
Mirrors matchmaker/models/published/ecai20_tk.py."""
from __future__ import annotations

import math
from typing import List, Optional

import torch
import torch.nn as nn

from .. import autograd, interaction


def sinusoid_position_features(dimensions: int, max_length: int, min_timescale: float = 1.0,
                               max_timescale: float = 1.0e4) -> torch.Tensor:
    """[1, max_length, dimensions] timing signal: sin half then cos half over geometrically spaced
    timescales (ecai20_tk.py:145-194)."""
    n_scales = dimensions // 2
    pos = torch.arange(max_length, dtype=torch.float32)
    step = math.log(float(max_timescale) / float(min_timescale)) / float(n_scales - 1)
    inv = min_timescale * torch.exp(torch.arange(n_scales, dtype=torch.float32) * -step)
    ang = pos.unsqueeze(1) * inv.unsqueeze(0)
    feats = torch.cat([torch.sin(ang), torch.cos(ang)], dim=1)
    if dimensions % 2:
        feats = torch.cat([feats, feats.new_zeros(max_length, 1)], dim=1)
    return feats.unsqueeze(0)


class ECAI20_TK(nn.Module):
    """forward(query_embeddings, document_embeddings, query_mask, document_mask,
    output_secondary_output=False) -> score [B] (ecai20_tk.py:87-131).

    State-dict keys match the reference: buffers ``mu``, ``sigma``, ``positional_features_q/_d``; parameters
    ``mixer``, ``kernel_bin_weights.weight``, ``kernel_alpha_scaler``, ``contextualizer.layers.*``."""

    @staticmethod
    def from_config(config, word_embeddings_out_dim):
        return ECAI20_TK(word_embeddings_out_dim,
                         kernels_mu=config["tk_kernels_mu"], kernels_sigma=config["tk_kernels_sigma"],
                         att_heads=config["tk_att_heads"], att_layer=config["tk_att_layer"],
                         att_ff_dim=config["tk_att_ff_dim"], max_length=config["max_doc_length"],
                         use_diff_posencoding=config["tk_use_diff_posencoding"],
                         mix_hybrid_context=config["tk_mix_hybrid_context"])

    def __init__(self, _embsize: int, kernels_mu: List[float], kernels_sigma: List[float], att_heads: int,
                 att_layer: int, att_ff_dim: int, max_length: int, use_diff_posencoding: bool,
                 mix_hybrid_context: bool):
        super().__init__()
        if len(kernels_mu) != len(kernels_sigma):
            raise Exception("len(kernels_mu) != len(kernels_sigma)")
        n_kernels = len(kernels_mu)
        self.use_diff_posencoding = use_diff_posencoding
        self.register_buffer("positional_features_q", sinusoid_position_features(_embsize, max_length))
        if use_diff_posencoding:
            self.register_buffer("positional_features_d",
                                 sinusoid_position_features(_embsize, max_length + 500)[:, 500:, :])
        else:
            self.register_buffer("positional_features_d", self.positional_features_q)
        layer = nn.TransformerEncoderLayer(_embsize, att_heads, dim_feedforward=att_ff_dim, dropout=0)
        self.contextualizer = nn.TransformerEncoder(layer, att_layer, norm=None, enable_nested_tensor=False)
        self.mix_hybrid_context = mix_hybrid_context
        self.mixer = nn.Parameter(torch.full([1], 0.5, dtype=torch.float32, requires_grad=True))
        self.register_buffer("mu", torch.tensor(kernels_mu, dtype=torch.float32).view(1, 1, 1, n_kernels))
        self.register_buffer("sigma", torch.tensor(kernels_sigma, dtype=torch.float32).view(1, 1, 1, n_kernels))
        self.kernel_bin_weights = nn.Linear(n_kernels, 1, bias=False)
        torch.nn.init.uniform_(self.kernel_bin_weights.weight, -0.014, 0.014)
        self.kernel_alpha_scaler = nn.Parameter(torch.full([1, 1, n_kernels], 1, dtype=torch.float32, requires_grad=True))

    def forward(self, query_embeddings: torch.Tensor, document_embeddings: torch.Tensor, query_mask: torch.Tensor,
                document_mask: torch.Tensor, output_secondary_output: bool = False):
        query_embeddings = self.forward_representation(
            query_embeddings, query_mask, self.positional_features_q[:, :query_embeddings.shape[1], :])
        document_embeddings = self.forward_representation(
            document_embeddings, document_mask, self.positional_features_d[:, :document_embeddings.shape[1], :])
        score, per_kernel = self.score_contextualized(query_embeddings, document_embeddings, query_mask, document_mask)
        if not output_secondary_output:
            return score
        with torch.no_grad():
            cos = interaction.kernel_pool(query_embeddings, document_embeddings, query_mask, document_mask, self.mu,
                                          self.sigma, self.kernel_bin_weights.weight, self.kernel_alpha_scaler, 1.0,
                                          want_cosine=True)["cosine"]
        query_mean_vector = query_embeddings.sum(dim=1) / query_mask.sum(dim=1).unsqueeze(-1)
        return score, {"score": score, "per_kernel": per_kernel, "query_mean_vector": query_mean_vector,
                       "cosine_matrix": cos}

    def score_contextualized(self, query_ctx, document_ctx, query_mask, document_mask):
        """The interaction stage alone (ecai20_tk.py:105-124): cosine -> RBF kernels -> masked sums -> log
        -> linear, one kernel launch forward, one backward."""
        return autograd.kernel_pool(query_ctx, document_ctx, query_mask, document_mask, self.mu, self.sigma,
                                    self.kernel_bin_weights.weight, self.kernel_alpha_scaler, 1.0)

    @torch.no_grad()
    def encode_documents(self, document_embeddings: torch.Tensor, document_mask: torch.Tensor):
        """The document side of ``forward`` (ecai20_tk.py:93-103), which does not depend on the query, for a store that
        is encoded once: (rows [n_live, D] fp32, the contextualised embeddings of the unmasked terms in passage order,
        lengths [B] int64).  ``score_store`` over them gives ``forward``'s scores."""
        ctx = self.forward_representation(document_embeddings, document_mask,
                                          self.positional_features_d[:, :document_embeddings.shape[1], :])
        live = document_mask.bool()
        return ctx[live].float().contiguous(), live.sum(dim=1)

    def score_store(self, query_ctx: torch.Tensor, query_mask: torch.Tensor, store: torch.Tensor,
                    doc_offsets: torch.Tensor, pair_q: torch.Tensor, pair_d: torch.Tensor,
                    max_doc_len: Optional[int] = None) -> torch.Tensor:
        """The counterpart of ``score_contextualized`` over rows from ``encode_documents`` (inference): pair p scores
        query ``pair_q[p]`` of query_ctx [n_q, Lq, D] against passage ``pair_d[p]``, rows ``doc_offsets[d] :
        doc_offsets[d+1]`` of store (see ``interaction.kernel_pool_store``)."""
        return interaction.kernel_pool_store(query_ctx, query_mask, store, doc_offsets, pair_q, pair_d, self.mu,
                                             self.sigma, self.kernel_bin_weights.weight, self.kernel_alpha_scaler, 1.0,
                                             max_doc_len=max_doc_len)

    def forward_representation(self, sequence_embeddings: torch.Tensor, sequence_mask: torch.Tensor,
                               positional_features=None) -> torch.Tensor:
        if positional_features is None:
            positional_features = self.positional_features_d[:, :sequence_embeddings.shape[1], :]
        ctx = self.contextualizer((sequence_embeddings + positional_features).transpose(1, 0),
                                  src_key_padding_mask=~sequence_mask.bool()).transpose(1, 0)
        if self.mix_hybrid_context:
            return self.mixer * sequence_embeddings + (1 - self.mixer) * ctx
        return ctx

    def get_param_stats(self):
        return ("TK: kernel_bin_weights: " + str(self.kernel_bin_weights.weight.data) + " kernel_alpha_scaler: " +
                str(self.kernel_alpha_scaler.data) + " mixer: " + str(self.mixer.data))

    def get_param_secondary(self):
        return {"kernel_bin_weights": self.kernel_bin_weights.weight,
                "kernel_alpha_scaler": self.kernel_alpha_scaler, "mixer": self.mixer}
