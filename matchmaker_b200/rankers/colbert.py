"""ColBERT with the late-interaction max-sim on the GPU kernel.  Mirrors matchmaker/models/colbert.py.

The BERT encoder + linear compressor stay ordinary PyTorch / HuggingFace modules, exactly as in the
reference; only the scoring lines (colbert.py:68-75, :100-112, :154-162) are replaced."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Union

import torch
from torch import nn

from .. import autograd, interaction


@dataclass
class ColBERTConfig:
    """Field-for-field the reference's ColBERTConfig (colbert.py:10-16), as a plain dataclass (the
    reference subclasses transformers.PretrainedConfig, which transformers >= 5 rejects for
    un-defaulted annotated fields)."""
    bert_model: Union[str, nn.Module] = "distilbert-base-uncased"
    compression_dim: int = 768
    dropout: float = 0.0
    return_vecs: bool = False
    trainable: bool = True
    model_type: str = "ColBERT"


class ColBERT(nn.Module):
    """forward(query: {"input_ids","attention_mask"}, document: {...}, use_fp16=True,
    output_secondary_output=False) -> score [B] (or (score, q_vecs, d_vecs) / (score, {}) as in the
    reference, colbert.py:54-86).  State-dict keys: ``bert_model.*``, ``compressor.{weight,bias}``."""

    is_teacher_model = False  # overridden by the dynamic-teacher runner (dynamic_teacher.py:174)

    @staticmethod
    def from_config(config):
        cfg = ColBERTConfig()
        cfg.bert_model = config["bert_pretrained_model"]
        cfg.compression_dim = config["colbert_compression_dim"]
        cfg.return_vecs = config.get("in_batch_negatives", False)
        cfg.trainable = config["bert_trainable"]
        return ColBERT(cfg)

    def __init__(self, cfg: ColBERTConfig) -> None:
        super().__init__()
        self.config = cfg
        self.return_vecs = cfg.return_vecs
        if isinstance(cfg.bert_model, str):
            from transformers import AutoModel
            self.bert_model = AutoModel.from_pretrained(cfg.bert_model)
        else:
            self.bert_model = cfg.bert_model  # any module returning (last_hidden_state, ...) with .config.hidden_size
        for p in self.bert_model.parameters():
            p.requires_grad = cfg.trainable
        self._dropout = torch.nn.Dropout(p=cfg.dropout)
        self.compressor = torch.nn.Linear(self.bert_model.config.hidden_size, cfg.compression_dim)

    def forward(self, query: Dict[str, torch.LongTensor], document: Dict[str, torch.LongTensor],
                use_fp16: bool = True, output_secondary_output: bool = False):
        with torch.autocast("cuda", enabled=use_fp16):
            query_vecs = self.forward_representation(query)
            document_vecs = self.forward_representation(document)
        score = self.score_vectors(query_vecs, document_vecs, query["attention_mask"], document["attention_mask"])
        if use_fp16:
            score = score.to(query_vecs.dtype)  # the reference's bmm/max/sum run under autocast
        if self.is_teacher_model:
            return (score, query_vecs, document_vecs)
        if self.return_vecs:
            score = (score, query_vecs, document_vecs)
        if output_secondary_output:
            return score, {}
        return score

    @staticmethod
    def score_vectors(query_vecs, document_vecs, query_mask, document_mask):
        """colbert.py:68-75 on the kernel: masked max over document tokens, sum over query tokens."""
        if query_vecs.dtype != document_vecs.dtype:
            document_vecs = document_vecs.to(query_vecs.dtype)
        return autograd.maxsim(query_vecs, document_vecs, query_mask, document_mask)

    def forward_representation(self, tokens: Dict[str, torch.LongTensor], sequence_type=None) -> torch.Tensor:
        vecs = self.bert_model(**tokens)[0]
        vecs = self.compressor(vecs)
        if sequence_type == "doc_encode" or sequence_type == "query_encode":
            vecs = vecs * tokens["attention_mask"].unsqueeze(-1)
        return vecs

    def forward_aggregation(self, query_vecs, document_vecs):
        """Unmasked pair aggregation (colbert.py:100-112); relies on zeroed padding vectors."""
        if query_vecs.dtype != document_vecs.dtype:
            document_vecs = document_vecs.to(query_vecs.dtype)
        return interaction.maxsim(query_vecs.contiguous(), document_vecs.contiguous())

    def forward_inbatch_aggregation(self, query_vecs, query_mask, document_vecs, document_mask,
                                    reference_mask_indexing: bool = True):
        """All-pairs scores [Nq, Nd] (colbert.py:154-162).  By default bit-compatible with the reference,
        including its indexing of ``document_mask`` by the query position (colbert.py:158; see DESIGN.md);
        pass ``reference_mask_indexing=False`` to mask every document with its own mask.  Differentiable: the
        scores train the encoder (in-batch negatives)."""
        if query_vecs.dtype != document_vecs.dtype:
            document_vecs = document_vecs.to(query_vecs.dtype)
        return autograd.maxsim_allpairs(query_vecs, query_mask, document_vecs, document_mask,
                                        reference_mask_indexing=reference_mask_indexing)

    def get_param_stats(self):
        return "ColBERT: / "

    def get_param_secondary(self):
        return {}
