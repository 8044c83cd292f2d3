"""Drop-in counterparts of the reference's interaction models (``matchmaker/models``): same class names,
constructor / ``from_config`` keys, ``forward`` signatures, state-dict keys and secondary-output keys; the
interaction arithmetic runs in the sm_90a kernels (``libmatchmaker_b200.so``), everything upstream of it
(embeddings, transformer / BERT encoders) stays ordinary PyTorch exactly as in the reference.

    reference                                        here
    matchmaker/models/knrm.py              KNRM        rankers.knrm.KNRM
    matchmaker/models/published/ecai20_tk.py ECAI20_TK rankers.tk.ECAI20_TK
    matchmaker/models/published/sigir20_tkl.py TKL_sigir20 rankers.tkl.TKL_sigir20
    matchmaker/models/colbert.py           ColBERT     rankers.colbert.ColBERT
    matchmaker/models/bert_dot.py          BERT_Dot    rankers.bert_dot.BERT_Dot
    matchmaker/models/published/cikm20_tk_sparse.py CIKM20_TK_Sparse rankers.tk_sparse.CIKM20_TK_Sparse
    matchmaker/models/conv_knrm.py         Conv_KNRM   rankers.conv_knrm.Conv_KNRM
"""
from .knrm import KNRM  # noqa: F401
from .tk import ECAI20_TK  # noqa: F401


def get_model_class(name: str):
    """The ``config["model"]`` strings of matchmaker/models/all.py:141-184 for the hot-path models."""
    from . import bert_dot, colbert, conv_knrm, tk_sparse, tkl
    table = {"knrm": KNRM, "TK": ECAI20_TK, "TKL": tkl.TKL_sigir20, "ColBERT": colbert.ColBERT,
             "bert_dot": bert_dot.BERT_Dot, "bert_tower": bert_dot.BERT_Dot,
             "TK_Sparse": tk_sparse.CIKM20_TK_Sparse, "conv_knrm": conv_knrm.Conv_KNRM}
    if name not in table:
        raise KeyError(f"model {name!r} is outside the interaction-scoring hot path covered by matchmaker_b200")
    return table[name]
