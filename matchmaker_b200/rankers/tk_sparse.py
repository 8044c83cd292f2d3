"""TK-Sparse (CIKM'20): TK plus a learned per-document-term gate that multiplies every kernel activation of its term.
Mirrors matchmaker/models/published/cikm20_tk_sparse.py; the interaction stage (:106-145) runs in the kernel-pooling
kernels with the gate applied inside the activation sum (one more exponent term per document row, no extra pass)."""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn

from .. import autograd, interaction
from .tk import sinusoid_position_features


class CIKM20_TK_Sparse(nn.Module):
    """forward(query_embeddings, document_embeddings, query_mask, document_mask, output_secondary_output=False)
    -> (score [B], document_stop_words [B,1,Ld])  (cikm20_tk_sparse.py:92-152: the reference returns the gate as well,
    train.py uses it for the L1 sparsity loss).

    State-dict keys as in the reference: ``mixer_stop``, ``mixer``, ``positional_features_q/_d``, ``mu``, ``sigma``,
    ``contextualizer.*``, ``kernel_bin_weights.weight``, ``kernel_alpha_scaler``, ``stop_word_reducer.*``,
    ``stop_word_reducer2.*``."""

    @staticmethod
    def from_config(config, word_embeddings_out_dim):
        return CIKM20_TK_Sparse(word_embeddings_out_dim, kernels_mu=config["tk_kernels_mu"],
                                kernels_sigma=config["tk_kernels_sigma"], att_heads=config["tk_att_heads"],
                                att_layer=config["tk_att_layer"], att_proj_dim=config["tk_att_proj_dim"],
                                att_ff_dim=config["tk_att_ff_dim"], max_length=config["max_doc_length"],
                                use_diff_posencoding=config["tk_use_diff_posencoding"])

    def __init__(self, _embsize: int, kernels_mu: List[float], kernels_sigma: List[float], att_heads: int, att_layer: int,
                 att_proj_dim: int, att_ff_dim: int, max_length: int, use_diff_posencoding: bool):
        super().__init__()
        if len(kernels_mu) != len(kernels_sigma):
            raise Exception("len(kernels_mu) != len(kernels_sigma)")
        n_kernels = len(kernels_mu)
        self.mixer_stop = nn.Parameter(torch.full([1], 0.5, dtype=torch.float32, requires_grad=True))
        self.mixer = nn.Parameter(torch.full([1], 0.5, dtype=torch.float32, requires_grad=True))
        self.use_diff_posencoding = use_diff_posencoding
        self.register_buffer("positional_features_q", sinusoid_position_features(_embsize, max_length))
        if use_diff_posencoding:
            self.register_buffer("positional_features_d", sinusoid_position_features(_embsize, max_length + 500)[:, 500:, :])
        else:
            self.register_buffer("positional_features_d", self.positional_features_q)
        layer = nn.TransformerEncoderLayer(_embsize, att_heads, dim_feedforward=att_ff_dim, dropout=0)
        self.contextualizer = nn.TransformerEncoder(layer, att_layer, norm=None, enable_nested_tensor=False)
        self.register_buffer("mu", torch.tensor(kernels_mu, dtype=torch.float32).view(1, 1, 1, n_kernels))
        self.register_buffer("sigma", torch.tensor(kernels_sigma, dtype=torch.float32).view(1, 1, 1, n_kernels))
        self.kernel_bin_weights = nn.Linear(n_kernels, 1, bias=False)
        torch.nn.init.uniform_(self.kernel_bin_weights.weight, -0.014, 0.014)
        self.kernel_alpha_scaler = nn.Parameter(torch.full([1, 1, n_kernels], 1, dtype=torch.float32, requires_grad=True))
        self.stop_word_reducer = nn.Linear(_embsize, 100, bias=True)
        self.stop_word_reducer2 = nn.Linear(100, 1, bias=True)
        torch.nn.init.constant_(self.stop_word_reducer2.bias, 1)

    def reanimate(self, added_bias):
        self.stop_word_reducer2.bias.data += added_bias

    def forward(self, query_embeddings: torch.Tensor, document_embeddings: torch.Tensor, query_mask: torch.Tensor,
                document_mask: torch.Tensor, output_secondary_output: bool = False):
        query_ctx, _ = self.forward_representation(query_embeddings, query_mask,
                                                   self.positional_features_q[:, :query_embeddings.shape[1], :])
        document_embeddings_orig = document_embeddings
        document_ctx, document_context_only = self.forward_representation(
            document_embeddings, document_mask, self.positional_features_d[:, :document_embeddings.shape[1], :])
        # the sparsity gate (:132-133) is a small MLP on [B, Ld, D]: ordinary PyTorch, as upstream of the interaction
        stop_in = self.mixer_stop * document_embeddings_orig + (1 - self.mixer_stop) * document_context_only
        document_stop_words = torch.nn.functional.relu(
            self.stop_word_reducer2(torch.tanh(self.stop_word_reducer(stop_in))).unsqueeze(1).squeeze(-1)) \
            * document_mask.unsqueeze(1)
        score, per_kernel = autograd.kernel_pool(query_ctx, document_ctx, query_mask, document_mask, self.mu, self.sigma,
                                                 self.kernel_bin_weights.weight, self.kernel_alpha_scaler, 1.0,
                                                 doc_gate=document_stop_words.squeeze(1))
        if output_secondary_output:
            query_mean_vector = query_ctx.sum(dim=1) / query_mask.sum(dim=1).unsqueeze(-1)
            return score, {"score": score, "per_kernel": per_kernel, "query_mean_vector": query_mean_vector,
                           "document_stop_words": document_stop_words}, document_stop_words
        return score, document_stop_words

    @torch.no_grad()
    def encode_documents(self, document_embeddings: torch.Tensor, document_mask: torch.Tensor):
        """The document side of ``forward`` (cikm20_tk_sparse.py:104-135), which does not depend on the query, for a
        store that is encoded once: (rows [n_live, D] fp32, lengths [B] int64, gate [n_live] fp32).  A term whose gate is
        exactly 0 adds exactly 0 to every kernel sum of every query, so only terms with a nonzero gate are kept: rows
        are the mixed embeddings of those terms in passage order and gate their gate values.  A passage whose terms are all
        gated to 0 keeps its first term (gate 0): it scores what ``forward`` gives it, not the -inf of a passage without
        rows.  ``score_store`` over them gives ``forward``'s scores."""
        document_ctx, document_context_only = self.forward_representation(
            document_embeddings, document_mask, self.positional_features_d[:, :document_embeddings.shape[1], :])
        stop_in = self.mixer_stop * document_embeddings + (1 - self.mixer_stop) * document_context_only
        gate = torch.nn.functional.relu(self.stop_word_reducer2(torch.tanh(self.stop_word_reducer(stop_in))).squeeze(-1)) \
            * document_mask
        mask = document_mask.bool()
        live = mask & (gate != 0)
        all_gated = ~live.any(dim=1) & mask.any(dim=1)
        live[all_gated, mask[all_gated].float().argmax(dim=1)] = True
        return document_ctx[live].float().contiguous(), live.sum(dim=1), gate[live].float().contiguous()

    def score_store(self, query_ctx: torch.Tensor, query_mask: torch.Tensor, store: torch.Tensor,
                    doc_offsets: torch.Tensor, pair_q: torch.Tensor, pair_d: torch.Tensor, gate: torch.Tensor,
                    max_doc_len: Optional[int] = None) -> torch.Tensor:
        """The interaction stage of ``forward`` over rows and gates from ``encode_documents`` (inference): pair p scores
        query ``pair_q[p]`` of query_ctx [n_q, Lq, D] against passage ``pair_d[p]``, rows ``doc_offsets[d] :
        doc_offsets[d+1]`` of store with their gate (see ``interaction.kernel_pool_store``)."""
        return interaction.kernel_pool_store(query_ctx, query_mask, store, doc_offsets, pair_q, pair_d, self.mu,
                                             self.sigma, self.kernel_bin_weights.weight, self.kernel_alpha_scaler, 1.0,
                                             max_doc_len=max_doc_len, gate=gate)

    def forward_representation(self, sequence_embeddings: torch.Tensor, sequence_mask: torch.Tensor, positional_features=None):
        """Returns (mixed embeddings, context-only embeddings) as cikm20_tk_sparse.py:154-169."""
        if positional_features is None:
            positional_features = self.positional_features_d[:, :sequence_embeddings.shape[1], :]
        sequence_embeddings = sequence_embeddings * sequence_mask.unsqueeze(-1)
        ctx = self.contextualizer((sequence_embeddings + positional_features).transpose(1, 0),
                                  src_key_padding_mask=~sequence_mask.bool()).transpose(1, 0)
        mixed = (self.mixer * sequence_embeddings + (1 - self.mixer) * ctx) * sequence_mask.unsqueeze(-1)
        return mixed, ctx

    def get_param_stats(self):
        return ("TK-Sparse: kernel_bin_weights: " + str(self.kernel_bin_weights.weight.data) + " kernel_alpha_scaler: " +
                str(self.kernel_alpha_scaler.data) + " mixer: " + str(self.mixer.data) + " mixer_stop: " + str(self.mixer_stop.data))

    def get_param_secondary(self):
        return {"kernel_bin_weights": self.kernel_bin_weights.weight, "kernel_alpha_scaler": self.kernel_alpha_scaler,
                "mixer": self.mixer, "mixer_stop": self.mixer_stop}
