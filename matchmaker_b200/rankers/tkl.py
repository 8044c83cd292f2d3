"""TKL (SIGIR'20, long documents): chunked transformer contextualisation in PyTorch + the interaction stage
(per-chunk cosine/RBF kernels, sliding-window pooling, saturation, top-3 windows) on the GPU kernels.
Mirrors matchmaker/models/published/sigir20_tkl.py.

Forward and backward of the interaction stage are CUDA kernels (``autograd.tkl_interaction``); gradients reach the
transformer, the kernel weights and the saturation parameters exactly as through the reference's eager op chain."""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn

from .. import autograd, interaction
from .tk import sinusoid_position_features


def chunk_documents(document_embeddings: torch.Tensor, document_mask: torch.Tensor, chunk_size: int = 40,
                    overlap: int = 5):
    """Pad (5 left, >= 10 right), unfold into extended chunks of 50 at stride 40, and mark the chunks whose 40
    centre positions hold at least one real token (sigir20_tkl.py:142-162).  Returns (chunks [B*C,50,D],
    chunk masks [B*C,50], packed [B*C] bool, C)."""
    ext = chunk_size + 2 * overlap
    ld = document_mask.shape[1]
    needed = ext - ((ld - overlap) % chunk_size) if ld > overlap else ext - overlap - ld
    emb = nn.functional.pad(document_embeddings, (0, 0, overlap, needed))
    msk = nn.functional.pad(document_mask, (overlap, needed))
    chunks = emb.unfold(1, ext, chunk_size).transpose(-1, -2)
    cmask = msk.unfold(1, ext, chunk_size)
    pieces = chunks.shape[1]
    chunks2 = chunks.reshape(-1, ext, emb.shape[-1])
    cmask2 = cmask.reshape(-1, ext)
    packed = cmask2[:, overlap:-overlap].sum(-1) != 0
    return chunks2, cmask2, packed, pieces


def chunk_slots(doc_length: int, chunk_size: int = 40, overlap: int = 5) -> int:
    """Chunk slots C of a document padded to doc_length positions: the ``pieces`` of :func:`chunk_documents`."""
    ext = chunk_size + 2 * overlap
    needed = ext - ((doc_length - overlap) % chunk_size) if doc_length > overlap else ext - overlap - doc_length
    return (overlap + doc_length + needed - ext) // chunk_size + 1


class TKL_sigir20(nn.Module):
    """forward(query_embeddings, document_embeddings, query_pad_oov_mask, document_pad_oov_mask,
    output_secondary_output=False) -> score [B] (sigir20_tkl.py:128-294).  Parameter names / shapes match the
    reference so its checkpoints load with ``load_state_dict``."""

    @staticmethod
    def from_config(config, word_embeddings_out_dim):
        return TKL_sigir20(word_embeddings_out_dim,
                           kernels_mu=config["tk_kernels_mu"], kernels_sigma=config["tk_kernels_sigma"],
                           att_heads=config["tk_att_heads"], att_layer=config["tk_att_layer"],
                           att_ff_dim=config["tk_att_ff_dim"], max_length=config["max_doc_length"],
                           use_pos_encoding=config["tk_use_pos_encoding"],
                           use_diff_posencoding=config["tk_use_diff_posencoding"],
                           saturation_type=config["tk_saturation_type"])

    def __init__(self, _embsize: int, kernels_mu: List[float], kernels_sigma: List[float], att_heads: int,
                 att_layer: int, att_ff_dim: int, max_length, use_pos_encoding, use_diff_posencoding,
                 saturation_type):
        super().__init__()
        if len(kernels_mu) != len(kernels_sigma):
            raise Exception("len(kernels_mu) != len(kernels_sigma)")
        if saturation_type not in ("embedding", "log"):
            # the reference's "idf" / "linear" branches read an undefined `query_idfs` (sigir20_tkl.py:215,237)
            raise ValueError("tk_saturation_type must be 'embedding' or 'log' (the other reference branches are dead code)")
        n_kernels = len(kernels_mu)
        self.max_length = max_length
        self.use_pos_encoding = use_pos_encoding
        self.use_diff_posencoding = use_diff_posencoding
        self.re_use_encoding = True
        self.chunk_size = 40
        self.overlap = 5
        self.extended_chunk_size = self.chunk_size + 2 * self.overlap
        self.sliding_window_size = 30
        self.top_k_chunks = 3
        self.saturation_type = saturation_type

        self.mu = nn.Parameter(torch.tensor(kernels_mu, dtype=torch.float32), requires_grad=False)
        self.sigma = nn.Parameter(torch.tensor(kernels_sigma, dtype=torch.float32), requires_grad=False)
        self.positional_features_q = nn.Parameter(sinusoid_position_features(_embsize, 30))
        if use_diff_posencoding:
            self.positional_features_d = nn.Parameter(
                sinusoid_position_features(_embsize, 2000 + 500 + self.extended_chunk_size)[:, 500:, :].clone())
        else:
            self.positional_features_d = self.positional_features_q
        self.mixer = nn.Parameter(torch.full([1], 0.5, dtype=torch.float32))
        self.mixer_sat = nn.Parameter(torch.full([1], 0.5, dtype=torch.float32))
        layer = nn.TransformerEncoderLayer(_embsize, att_heads, dim_feedforward=att_ff_dim, dropout=0)
        self.contextualizer = nn.TransformerEncoder(layer, att_layer, norm=None, enable_nested_tensor=False)

        def sat_linear():
            lin = nn.Linear(2, 1, bias=True)
            torch.nn.init.constant_(lin.bias, 100)
            torch.nn.init.uniform_(lin.weight, -0.014, 0.014)
            return lin

        self.saturation_linear = sat_linear()
        self.saturation_linear2 = sat_linear()
        self.saturation_linear3 = sat_linear()
        self.sat_normer = nn.LayerNorm(2, elementwise_affine=True)
        self.sat_emb_reduce1 = nn.Linear(_embsize, 1, bias=False)
        self.kernel_mult = nn.Parameter(torch.full([4, 1, 1, 1, n_kernels], 1, dtype=torch.float32))
        self.chunk_scoring = nn.Parameter(torch.full([1, self.top_k_chunks * 5], 1, dtype=torch.float32))
        self.mixer_end = nn.Parameter(torch.full([1], 0.5, dtype=torch.float32))
        self.dense = nn.Linear(n_kernels, 1, bias=False)
        torch.nn.init.uniform_(self.dense.weight, -0.014, 0.014)

    # -- chunking (sigir20_tkl.py:142-162) -----------------------------------------------------
    def chunk_documents(self, document_embeddings: torch.Tensor, document_mask: torch.Tensor):
        return chunk_documents(document_embeddings, document_mask, self.chunk_size, self.overlap)

    def _saturation_params(self):
        if self.saturation_type == "embedding":
            p = torch.cat([self.sat_normer.weight, self.sat_normer.bias,
                           self.saturation_linear.weight.view(-1), self.saturation_linear.bias,
                           self.saturation_linear2.weight.view(-1), self.saturation_linear2.bias,
                           self.saturation_linear3.weight.view(-1), self.saturation_linear3.bias])
            return p, self.sat_emb_reduce1.weight.view(-1)
        return self.kernel_mult[0].reshape(-1), None

    def forward(self, query_embeddings: torch.Tensor, document_embeddings: torch.Tensor,
                query_pad_oov_mask: torch.Tensor, document_pad_oov_mask: torch.Tensor,
                output_secondary_output: bool = False):
        query_ctx, _ = self.forward_representation(
            query_embeddings, query_pad_oov_mask, self.positional_features_q[:, :query_embeddings.shape[1], :])
        chunks2, cmask2, packed, pieces = self.chunk_documents(document_embeddings, document_pad_oov_mask)
        docs_packed = chunks2[packed]
        pad_packed = cmask2[packed]
        docs_ctx, _ = self.forward_representation(docs_packed, pad_packed,
                                                  self.positional_features_d[:, :docs_packed.shape[1], :])
        doc_chunks = docs_ctx[:, self.overlap:-self.overlap, :]
        chunk_mask = pad_packed[:, self.overlap:-self.overlap]

        sat_params, sat_red = self._saturation_params()
        score, orig_score, top_idx, top15 = autograd.tkl_interaction(
            query_ctx, query_pad_oov_mask, doc_chunks.contiguous(), chunk_mask.contiguous(), packed, pieces, self.mu,
            self.sigma, self.dense.weight, self.saturation_type, sat_params, sat_red, self.chunk_scoring)
        if not output_secondary_output:
            return score
        return score, {"score": score, "orig_score": orig_score, "top_non_overlapping_idx": top_idx,
                       "orig_doc_len": document_pad_oov_mask.sum(dim=-1), "top_k_non_overlapping": top15,
                       "total_chunks": chunks2.shape[0], "packed_chunks": docs_packed.shape[0]}

    @torch.no_grad()
    def encode_documents(self, document_embeddings: torch.Tensor, document_mask: torch.Tensor):
        """The document half of ``forward`` (sigir20_tkl.py:142-175) for a store that is encoded once: chunking,
        packing, the transformer over every packed chunk (alone, with the same positions) and the overlap trim.  None of
        it depends on the query or on the rest of the batch.  Returns (chunks [n_packed, 40, D] fp32, chunk masks
        [n_packed, 40], the slot of every chunk within its passage [n_packed] int64, packed chunks per passage [B]
        int64), passages in batch order and each passage's chunks in slot order.  ``score_store`` over them gives what
        ``forward`` gives the passages padded to any length at least as long as them."""
        chunks2, cmask2, packed, pieces = self.chunk_documents(document_embeddings, document_mask)
        docs_packed = chunks2[packed]
        pad_packed = cmask2[packed]
        docs_ctx, _ = self.forward_representation(docs_packed, pad_packed,
                                                  self.positional_features_d[:, :docs_packed.shape[1], :])
        chunks = docs_ctx[:, self.overlap:-self.overlap, :].float().contiguous()
        chunk_mask = pad_packed[:, self.overlap:-self.overlap].contiguous()
        slots = torch.arange(packed.numel(), device=packed.device)[packed] % pieces
        return chunks, chunk_mask, slots, packed.view(-1, pieces).sum(dim=1)

    @torch.no_grad()
    def score_store(self, query_ctx: torch.Tensor, query_mask: torch.Tensor, chunks: torch.Tensor,
                    chunk_mask: torch.Tensor, doc_slots: torch.Tensor, pair_q: torch.Tensor, pair_d: torch.Tensor,
                    output_secondary_output: bool = False):
        """The interaction stage of ``forward`` over chunks from ``encode_documents`` (inference): pair p scores query
        ``pair_q[p]`` of query_ctx [n_q, Lq, D] (``forward_representation`` with ``positional_features_q``) against the
        chunk slots ``doc_slots[pair_d[p]]`` (see ``interaction.tkl_store_window_scores``), then the top-3 windows.
        With ``output_secondary_output`` also returns ``forward``'s ``score`` / ``orig_score`` /
        ``top_non_overlapping_idx`` / ``top_k_non_overlapping`` entries: the selected regions of every pair."""
        sat_params, sat_red = self._saturation_params()
        window = interaction.tkl_store_window_scores(query_ctx, query_mask, chunks, chunk_mask, doc_slots, pair_q, pair_d,
                                                     self.mu, self.sigma, self.dense.weight, self.saturation_type,
                                                     sat_params, sat_red)
        score, orig_score, top_idx, top15 = interaction.tkl_top_hills(window, self.chunk_scoring)
        if not output_secondary_output:
            return score
        return score, {"score": score, "orig_score": orig_score, "top_non_overlapping_idx": top_idx,
                       "top_k_non_overlapping": top15}

    def forward_representation(self, sequence_embeddings: torch.Tensor, sequence_mask: torch.Tensor,
                               positional_features=None):
        pos_sequence = sequence_embeddings
        if self.use_pos_encoding:
            if positional_features is None:
                positional_features = self.positional_features_d[:, :sequence_embeddings.shape[1], :]
            pos_sequence = sequence_embeddings + positional_features
        ctx = self.contextualizer(pos_sequence.transpose(1, 0),
                                  src_key_padding_mask=~sequence_mask.bool()).transpose(1, 0)
        mixed = (self.mixer * sequence_embeddings + (1 - self.mixer) * ctx) * sequence_mask.unsqueeze(-1)
        return mixed, ctx

    def get_param_stats(self):
        return ("TK: dense w: " + str(self.dense.weight.data) + " self.chunk_scoring: " + str(self.chunk_scoring.data) +
                " self.kernel_mult: " + str(self.kernel_mult.data) + " mixer: " + str(self.mixer.data))

    def get_param_secondary(self):
        return {"dense_weight": self.dense.weight,
                "saturation_linear_weight": self.saturation_linear.weight,
                "saturation_linear_bias": self.saturation_linear.bias,
                "saturation_linear2_weight": self.saturation_linear2.weight,
                "saturation_linear2_bias": self.saturation_linear2.bias,
                "saturation_linear3_weight": self.saturation_linear3.weight,
                "saturation_linear3_bias": self.saturation_linear3.bias,
                "chunk_scoring": self.chunk_scoring, "kernel_mult": self.kernel_mult, "mixer": self.mixer}
