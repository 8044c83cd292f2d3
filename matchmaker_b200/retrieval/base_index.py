"""Mirror of matchmaker/retrieval/base_index.py: the interface dense_retrieval.py drives, and the per-rank plumbing the
GPU indexers share."""
import os
from typing import List, Optional

import numpy
import torch

from .. import _lib, sharding


class BaseNNIndexer:
    """prepare(data_chunks) / index(ids, data_chunks) / search(query_vec, top_n) -> (scores, ids)."""

    def __init__(self, config):
        self.token_dim = config["token_dim"]
        self.use_gpu = config["faiss_use_gpu"]
        self.use_fp16 = config["token_dtype"] == "float16"

    def prepare(self, data_chunks: List[numpy.ndarray], subsample=-1):
        pass

    def index(self, ids: List[numpy.ndarray], data_chunks: List[numpy.ndarray]):
        pass

    def search(self, query_vec: numpy.ndarray, top_n: int):
        pass


class GPUIndexer(BaseNNIndexer):
    """An indexer on one GPU per rank of a ``torch.distributed`` job (one rank without it): each rank indexes its
    share of the rows and saves it to a file of its own."""
    gpu_only = True   # False where the reference runs on the CPU whatever faiss_use_gpu says and this index ignores it

    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config)
        if self.gpu_only and not self.use_gpu:
            raise _lib.MatchmakerB200Error(f"{type(self).__name__} runs on the GPU only (faiss_use_gpu must be True); "
                                           "there is no CPU fallback")
        # token_dtype float16 -> fp16 storage (faiss useFloat16); anything else -> fp32 storage
        self.store_dtype = torch.float16 if self.use_fp16 else torch.float32
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.group = process_group

    def _world(self):
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank(self.group), dist.get_world_size(self.group)
        return 0, 1

    def _shard_path(self, path: str) -> str:
        """This rank's file: ``<path>.rank<r>of<w>`` with more than one rank (every rank owns different rows, so they
        must not write the same file)."""
        rank, world = self._world()
        return path if world == 1 else f"{path}.rank{rank}of{world}"

    def _load_shard(self, fn: str, row_range: bool = True) -> dict:
        """The index file fn of this rank, refused unless it was written by this rank of a job of this world size, for
        this rank's rows of its ``n_total`` (with ``row_range``) and for this token_dtype.  A file without the world /
        rank / lo / hi / token_dtype keys predates them: one rank, all rows, fp16."""
        rank, world = self._world()
        if not os.path.isfile(fn):
            raise _lib.MatchmakerB200Error(f"no index file {fn} for rank {rank} of {world}: re-index, or load with the "
                                           "world size the index was saved with")
        blob = torch.load(fn)
        saved_world = blob.get("world", blob.get("fingerprint", {}).get("world", 1))
        saved_rank = blob.get("rank", 0)
        held = needs = ""
        ok = saved_world == world and saved_rank == rank
        if row_range:
            lo, hi = sharding.shard_bounds(blob["n_total"], rank, world)
            saved = blob.get("lo", lo), blob.get("hi", hi)
            ok = ok and saved == (lo, hi)
            held, needs = f" holds rows [{saved[0]},{saved[1]}) of", f" and needs rows [{lo},{hi})"
        if not ok:
            raise _lib.MatchmakerB200Error(f"index file {fn}{held or ' was written by'} rank {saved_rank} of {saved_world}; "
                                           f"this job is rank {rank} of {world}{needs} -- re-index or load with the same "
                                           "world size")
        if blob.get("token_dtype", "torch.float16") != str(self.store_dtype):
            raise _lib.MatchmakerB200Error(f"index file was written with token_dtype {blob.get('token_dtype')}, this indexer "
                                           f"is configured for {self.store_dtype}")
        return blob
