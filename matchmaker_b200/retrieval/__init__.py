"""Index API of matchmaker/retrieval (base_index.py:4-32) on the H100 kernels: the exact inner-product index
(`faiss_index_type: "full"`, dense_retrieval.py:310-311), the inverted-file index (`faiss_index_type: "ivf"`), the
graph index (`faiss_index_type: "hnsw"`) and the anisotropic-hashing index (`faiss_index_type: "scann"`); TK /
TK-Sparse and TKL re-ranking over an encoded document store (`TKDocumentStore`, `TKLDocumentStore`)."""
from .base_index import BaseNNIndexer  # noqa: F401
from .flat_ip_index import FlatIPIndexer  # noqa: F401
from .ivf_index import IVFIndexer  # noqa: F401
from .graph_index import GraphIndexer  # noqa: F401
from .scann_index import ScaNNIndexer  # noqa: F401
from .colbert_rerank import ColBERTTokenIndex  # noqa: F401
from .colbert_e2e import ColBERTEndToEndIndexer  # noqa: F401
from .colbert_ivf import ColBERTIVFIndexer  # noqa: F401
from .colbert_residual import ColBERTResidualIndexer  # noqa: F401
from .tk_store import TKDocumentStore  # noqa: F401
from .tkl_store import TKLDocumentStore  # noqa: F401
