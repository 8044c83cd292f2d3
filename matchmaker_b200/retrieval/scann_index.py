"""Partitioned anisotropic-hashing (AH) index on the H100 kernels.

Drop-in for ``ScaNNIndexer`` (matchmaker/retrieval/scann_index.py:10-53), selected by ``faiss_index_type: "scann"`` in
dense_retrieval.py: same config keys (``token_dim``, ``token_dtype``, ``query_sets``: the build-time shortlist size is
``index_hit_top_n`` of the first query set, else its ``top_n``), same methods (training happens inside ``index()``;
``save`` / ``load`` take a directory), numpy in / numpy out.  ``faiss_use_gpu`` is ignored: the reference always runs
ScaNN on the CPU, this index always runs on the GPU.  Parity with ScaNN is not pinned; the settings below are this
project's reading of ``tree(num_leaves=sqrt(n), num_leaves_to_search=100).score_ah(2, 0.2).reorder(top_n)``.

- Leaves: nlist = int(sqrt(n)) unit centroids trained by IVFIndexer's spherical k-means (at most 256 training points
  per leaf, where ScaNN trains on all n); a query probes the min(100, nlist) leaves of best <q, centroid>.
- Codes: the residual r = x - c_leaf(x) (fp32) in M = dim / 2 blocks of 2 dimensions, 16 codewords per block, one
  codebook shared by all leaves, 4 bits per block: a row is dim / 4 bytes.  Codes and codebook minimise the anisotropic
  loss |e|^2 + (eta - 1) (e . x/|x|)^2 of the error e = r - r~, eta = (dim - 1) T^2 / (1 - T^2), T = 0.2: the error
  along the data point is what a query's score sees.
- Search: the probed leaves' codes are scanned through per-query lookup tables (interaction.ah_search) for a shortlist
  of kr = max(build-time top_n, top_n) rows, which are re-scored exactly from the stored rows (interaction.ah_reorder).

Multi-GPU: every rank is given the same chunks; rank 0 trains the centroids and the codebook and broadcasts them, each
rank codes its shard_bounds rows, and the per-rank top-k lists are merged with one all-gather.
"""
from __future__ import annotations

import math
import os
from typing import List, Optional

import numpy
import torch

from .. import _lib, interaction, sharding
from .base_index import GPUIndexer
from .ivf_index import IVFIndexer

AH_THRESHOLD = 0.2            # ScaNN's anisotropic_quantization_threshold
AH_TRAIN_SAMPLE = 100_000     # rows the codebook is trained on (ScaNN's score_ah default sample size)
AH_ROUNDS = 4                 # (assign, update) rounds after the isotropic start
AH_KMEANS_ITERATIONS = 10     # per-block isotropic k-means of the start
AH_ENCODE_SWEEPS = 2          # coordinate-descent sweeps over the blocks when every row is coded
AH_SEED = 4321
MAX_PROBE = 100               # ScaNN's num_leaves_to_search
_CHUNK = 1 << 16              # rows per step of the coding and of the least-squares accumulation
_NO_RESULT = -3.4028234663852886e38


def leaf_count(n: int) -> int:
    return max(1, int(math.sqrt(n)))


def probe_count(nlist: int) -> int:
    return min(MAX_PROBE, nlist)


def build_top_n(config) -> int:
    """The reference's build-time shortlist size: ``index_hit_top_n`` of the first query set, else its ``top_n``."""
    c = next(iter(config["query_sets"].values()))
    return int(c.get("index_hit_top_n", c["top_n"]))


def shortlist_size(build_n: int, top_n: int) -> int:
    """kr = max(build-time top_n, search top_n), within 1 <= kr <= 1024."""
    kr = max(int(build_n), int(top_n))
    if kr > interaction.AH_MAX_KR or min(int(build_n), int(top_n)) < 1:
        key = "index_hit_top_n" if int(build_n) >= int(top_n) else "top_n"
        raise _lib.MatchmakerB200Error(f"{key}: the AH shortlist max(index_hit_top_n or top_n, top_n) = {kr} must be in "
                                       f"[1, {interaction.AH_MAX_KR}]")
    return kr


def anisotropic_eta(dim: int, threshold: float = AH_THRESHOLD) -> float:
    """eta = (dim - 1) T^2 / (1 - T^2): the weight of the parallel error for a threshold T on <q, x> / |x|."""
    return (dim - 1) * threshold * threshold / (1.0 - threshold * threshold)


def pack_codes(codes: torch.Tensor) -> torch.Tensor:
    """[n, M] codes in 0..15 -> [n, M/2] uint8: block 2j in the low nibble of byte j, block 2j + 1 in the high one."""
    c = codes.to(torch.uint8)
    return (c[:, 0::2] | (c[:, 1::2] << 4)).contiguous()


def unpack_codes(packed: torch.Tensor) -> torch.Tensor:
    """Inverse of pack_codes: [n, M] int64."""
    p = packed.to(torch.int64)
    return torch.stack([p & 15, p >> 4], dim=2).reshape(p.shape[0], -1)


def unit_rows(x: torch.Tensor) -> torch.Tensor:
    """x / |x| per row in fp64, 0 for a zero row (which then has the plain squared loss)."""
    x = x.double()
    nrm = x.norm(dim=1, keepdim=True)
    return torch.where(nrm > 0, x / nrm.clamp_min(1e-300), torch.zeros_like(x))


def decode(codebook: torch.Tensor, codes: torch.Tensor) -> torch.Tensor:
    """r~ [n, dim] from codes [n, M] and a codebook [M, 16, 2]."""
    M = codebook.shape[0]
    return codebook[torch.arange(M, device=codes.device), codes].reshape(codes.shape[0], 2 * M)


def ah_loss(r: torch.Tensor, xhat: torch.Tensor, codebook: torch.Tensor, codes: torch.Tensor, eta: float) -> torch.Tensor:
    """Per-row anisotropic loss |e|^2 + (eta - 1) (e . xhat)^2, e = r - r~, in fp64."""
    e = r.double() - decode(codebook.double(), codes)
    return (e * e).sum(1) + (eta - 1.0) * (e * xhat.double()).sum(1) ** 2


def nearest_codes(r: torch.Tensor, codebook: torch.Tensor) -> torch.Tensor:
    """Isotropic coding: the nearest codeword of every block (lowest index on ties), [n, M] int64."""
    M = codebook.shape[0]
    out = torch.empty((r.shape[0], M), dtype=torch.int64, device=r.device)
    cb = codebook.double()
    for lo in range(0, r.shape[0], _CHUNK):
        rb = r[lo:lo + _CHUNK].double().view(-1, M, 1, 2)
        out[lo:lo + _CHUNK] = ((rb - cb.unsqueeze(0)) ** 2).sum(-1).argmin(-1)
    return out


def coordinate_descent(r: torch.Tensor, xhat: torch.Tensor, codebook: torch.Tensor, codes: torch.Tensor, eta: float,
                       sweeps: int) -> torch.Tensor:
    """`sweeps` passes over the blocks in ascending order: each block takes the codeword that minimises the full loss
    with the other blocks fixed (the current one unless another is strictly better), fp64.  Never raises a row's loss."""
    M = codebook.shape[0]
    cb = codebook.double()
    out = codes.clone()
    for lo in range(0, r.shape[0], _CHUNK):
        rb, xb = r[lo:lo + _CHUNK].double(), xhat[lo:lo + _CHUNK].double()
        cur = out[lo:lo + _CHUNK].clone()
        ar = torch.arange(rb.shape[0], device=r.device)
        for _ in range(sweeps):
            e = rb - decode(cb, cur)
            p = (e * xb).sum(1)
            for m in range(M):
                rm, xm = rb[:, 2 * m:2 * m + 2], xb[:, 2 * m:2 * m + 2]
                p_rest = p - (e[:, 2 * m:2 * m + 2] * xm).sum(1)
                cand = rm.unsqueeze(1) - cb[m].unsqueeze(0)                       # [b, 16, 2]
                par = p_rest.unsqueeze(1) + (cand * xm.unsqueeze(1)).sum(-1)
                loss = (cand * cand).sum(-1) + (eta - 1.0) * par * par
                best = loss.argmin(1)
                keep = loss[ar, best] >= loss[ar, cur[:, m]]
                j = torch.where(keep, cur[:, m], best)
                cur[:, m] = j
                e[:, 2 * m:2 * m + 2] = cand[ar, j]
                p = p_rest + (cand[ar, j] * xm).sum(1)
        out[lo:lo + _CHUNK] = cur
    return out


def block_kmeans(r: torch.Tensor, iterations: int = AH_KMEANS_ITERATIONS, seed: int = AH_SEED) -> torch.Tensor:
    """Per-block isotropic k-means with 16 centres, started from 16 seeded rows; an empty centre keeps its value.
    Sums run as fp64 matrix products, so the result is reproducible.  [M, 16, 2] fp64."""
    n, dim = r.shape
    M = dim // 2
    pts = r.double().view(n, M, 2).permute(1, 0, 2).contiguous()               # [M, n, 2]
    start = torch.from_numpy(numpy.random.RandomState(seed).permutation(n)[:16] % n).to(r.device)
    cb = pts[:, start, :].clone()
    if cb.shape[1] < 16:                                                       # fewer than 16 rows: repeat them
        cb = cb[:, torch.arange(16, device=r.device) % cb.shape[1]]
    step = max(1, (1 << 26) // max(1, n * 16))
    for _ in range(iterations):
        for m0 in range(0, M, step):
            p = pts[m0:m0 + step]
            c = cb[m0:m0 + step]
            a = ((p.unsqueeze(2) - c.unsqueeze(1)) ** 2).sum(-1).argmin(-1)
            oh = torch.nn.functional.one_hot(a, 16).double()                   # [mb, n, 16]
            sums = torch.bmm(oh.transpose(1, 2), p)
            cnt = oh.sum(1).unsqueeze(-1)
            cb[m0:m0 + step] = torch.where(cnt > 0, sums / cnt.clamp_min(1.0), c)
    return cb


def least_squares_codebook(r: torch.Tensor, xhat: torch.Tensor, codes: torch.Tensor, codebook: torch.Tensor,
                           eta: float) -> torch.Tensor:
    """The codebook minimising the summed anisotropic loss for fixed codes: normal equations over all 32 M codeword
    coordinates, (D + (eta - 1) U^T U) theta = R + (eta - 1) U^T (xhat . r), solved by Cholesky in fp64.  D counts the
    uses of every codeword, U scatters xhat into the slots of the used codewords.  An unused codeword keeps its value."""
    n, dim = r.shape
    M = dim // 2
    K = 32 * M
    dev = r.device
    G = torch.zeros((K, K), dtype=torch.float64, device=dev)
    rhs = torch.zeros(K, dtype=torch.float64, device=dev)
    cnt = torch.zeros((M, 16), dtype=torch.float64, device=dev)
    step = max(1, min(_CHUNK, (1 << 28) // (8 * K)))
    for lo in range(0, n, step):
        rb, xb, cb = r[lo:lo + step].double(), xhat[lo:lo + step].double(), codes[lo:lo + step]
        oh = torch.nn.functional.one_hot(cb, 16).double()                      # [b, M, 16]
        cnt += oh.sum(0)
        R = (oh.unsqueeze(-1) * rb.view(-1, M, 1, 2)).reshape(-1, K)
        U = (oh.unsqueeze(-1) * xb.view(-1, M, 1, 2)).reshape(-1, K)
        G += U.T @ U
        rhs += R.sum(0) + (eta - 1.0) * (U.T @ (xb * rb).sum(1))
    A = (eta - 1.0) * G
    d = cnt.unsqueeze(-1).expand(M, 16, 2).reshape(K)
    unused = d == 0
    A.diagonal().add_(torch.where(unused, torch.ones_like(d), d))
    rhs = torch.where(unused, codebook.double().reshape(K), rhs)
    L = torch.linalg.cholesky(A)
    return torch.cholesky_solve(rhs.unsqueeze(1), L).view(M, 16, 2)


def train_codebook(r: torch.Tensor, xhat: torch.Tensor, eta: float, rounds: int = AH_ROUNDS):
    """Isotropic start (block_kmeans, nearest codes), then `rounds` of (coordinate-descent assignment from the previous
    codes, least-squares update).  Returns (isotropic codebook, trained codebook [M, 16, 2] fp64, codes of the sample,
    mean loss at the start and after every round)."""
    iso = block_kmeans(r)
    codes = nearest_codes(r, iso)
    cb = iso
    losses = [float(ah_loss(r, xhat, cb, codes, eta).mean())]
    for _ in range(rounds):
        codes = coordinate_descent(r, xhat, cb, codes, eta, 1)
        cb = least_squares_codebook(r, xhat, codes, cb, eta)
        losses.append(float(ah_loss(r, xhat, cb, codes, eta).mean()))
    return iso, cb, codes, losses


def encode(r: torch.Tensor, xhat: torch.Tensor, codebook: torch.Tensor, eta: float,
           sweeps: int = AH_ENCODE_SWEEPS) -> torch.Tensor:
    """AH codes [n, M] int64 of residuals r: nearest codes, then `sweeps` coordinate-descent sweeps."""
    return coordinate_descent(r, xhat, codebook, nearest_codes(r, codebook), eta, sweeps)


class ScaNNIndexer(GPUIndexer):
    """faiss_index_type "scann" on the GPU.  ``faiss_use_gpu`` is read and ignored (see the module docstring)."""
    gpu_only = False

    def __init__(self, config, device: Optional[torch.device] = None, process_group=None):
        super().__init__(config, device, process_group)
        self.top_n = build_top_n(config)
        shortlist_size(self.top_n, 1)
        if int(self.token_dim) % 64:
            raise _lib.MatchmakerB200Error(f"token_dim = {self.token_dim}: the AH index needs a multiple of 64")
        self.eta = anisotropic_eta(int(self.token_dim))
        self.nlist = self.nprobe = 0
        self.ivf: Optional[IVFIndexer] = None            # leaves: centroids, layout
        self.codebook: Optional[torch.Tensor] = None     # [M, 16, 2] f32
        self.codebook_iso = None                         # the isotropic start of the training (rank 0)
        self.codes: Optional[torch.Tensor] = None        # [n_local, dim/4] uint8, leaf order
        self.rows: Optional[torch.Tensor] = None         # [n_local, dim] fp16 / fp32, leaf order
        self.ids: Optional[torch.Tensor] = None          # [n_local] int64
        self.list_offsets: Optional[torch.Tensor] = None
        self.max_list_len = 0
        self.n_total = 0
        self.train_loss: List[float] = []
        self.build_seconds = {}

    def _leaves(self, nlist: int, nprobe: int):
        self.nlist, self.nprobe = nlist, nprobe
        self.ivf = IVFIndexer({"token_dim": self.token_dim, "faiss_use_gpu": True,
                               "token_dtype": "float16" if self.use_fp16 else "float32",
                               "faiss_ivf_list_count": nlist, "faiss_ivf_search_probe_count": nprobe},
                              device=self.device, process_group=self.group)

    # ------------------------------------------------------------------ training
    def _sample(self, data_chunks, n: int) -> torch.Tensor:
        """A seeded sample of min(n, AH_TRAIN_SAMPLE) rows (in their order) in the storage dtype."""
        m = min(n, AH_TRAIN_SAMPLE)
        sel = numpy.sort(numpy.random.RandomState(AH_SEED).permutation(n)[:m])
        parts, off = [], 0
        for c in data_chunks:
            lo, hi = numpy.searchsorted(sel, [off, off + len(c)])
            if hi > lo:
                parts.append(torch.from_numpy(numpy.ascontiguousarray(numpy.asarray(c)[sel[lo:hi] - off])))
            off += len(c)
        return torch.cat(parts).to(self.device).to(self.store_dtype)

    def assign(self, x: torch.Tensor) -> torch.Tensor:
        """The leaf of every row of x [n, dim] (argmax <x, centroid>, lowest leaf on ties), [n] int64.  The coarse
        search runs _CHUNK rows at a time, so its scratch does not grow with n."""
        a = torch.empty(x.shape[0], dtype=torch.int64, device=x.device)
        for c0 in range(0, x.shape[0], _CHUNK):
            a[c0:c0 + _CHUNK] = interaction.flat_ip_topk(x[c0:c0 + _CHUNK], self.ivf.c_store, 1,
                                                         split_scale=self.ivf.c_scale)[1][:, 0]
        return a

    def train(self, data_chunks, n: int):
        """Rank 0's share of index(): the leaves (IVFIndexer.train) and the codebook, on the device."""
        import time
        torch.cuda.synchronize(self.device)
        t0 = time.perf_counter()
        cents = self.ivf.train(data_chunks)
        self.ivf.set_centroids(cents)
        torch.cuda.synchronize(self.device)
        t1 = time.perf_counter()
        x = self._sample(data_chunks, n)
        xf = x.float()
        r, xhat = xf - self.ivf.centroids[self.assign(x)], unit_rows(xf)
        del x, xf
        self.codebook_iso, cb, _, self.train_loss = train_codebook(r, xhat, self.eta)
        torch.cuda.synchronize(self.device)
        self.build_seconds.update(kmeans=t1 - t0, ah_training=time.perf_counter() - t1)
        return cents, cb.float()

    # ------------------------------------------------------------------ adding
    def index(self, ids: List[numpy.ndarray], data_chunks: List[numpy.ndarray]):
        """ids: list of int64 arrays; data_chunks: list of [n_i, token_dim] arrays.  Trains the leaves and the codebook
        (rank 0, broadcast), then codes this rank's rows shard_bounds(n, rank, world)."""
        from .token_storage import blocks_to_device
        rank, world = self._world()
        n = int(sum(len(x) for x in ids))
        if n < 1:
            raise _lib.MatchmakerB200Error("the AH index needs at least one row")
        self._leaves(leaf_count(n), probe_count(leaf_count(n)))
        M = int(self.token_dim) // 2
        if rank == 0:
            cents, cb = self.train(data_chunks, n)
        else:
            cents = torch.empty((self.nlist, self.token_dim), dtype=torch.float32, device=self.device)
            cb = torch.empty((M, 16, 2), dtype=torch.float32, device=self.device)
        if world > 1:
            import torch.distributed as dist
            dist.broadcast(cents, 0, group=self.group)
            dist.broadcast(cb, 0, group=self.group)
        self.ivf.set_centroids(cents)
        self.codebook = cb.contiguous()
        lo, hi = sharding.shard_bounds(n, rank, world)
        self.n_total, self.lo, self.hi = n, lo, hi
        if hi > lo:
            id_parts, off = [], 0
            for i_arr in ids:
                a, b = max(lo, off), min(hi, off + len(i_arr))
                if a < b:
                    id_parts.append(torch.from_numpy(numpy.ascontiguousarray(i_arr[a - off:b - off]).astype(numpy.int64)))
                off += len(i_arr)
            with torch.cuda.device(self.device):   # no reference kept here: add() replaces the rows by their sorted copy
                self.add(blocks_to_device(data_chunks, lo, hi, self.device).to(self.store_dtype),
                         torch.cat(id_parts).to(self.device))
        else:
            self.add(torch.empty((0, self.token_dim), dtype=self.store_dtype, device=self.device),
                     torch.empty(0, dtype=torch.int64, device=self.device))

    def add(self, vecs: torch.Tensor, ids: torch.Tensor):
        """Sort `vecs` into their leaves and code them (replaces the index content).  Needs the centroids and the
        codebook.  Besides the stored index (the sorted rows, codes, ids) and the caller's `vecs`, the device memory
        this takes is the leaf ids and their stable sort (tens of bytes per row) plus scratch bounded by _CHUNK rows: the assignment and
        the coding both run _CHUNK rows at a time."""
        import time
        torch.cuda.synchronize(self.device)
        t0 = time.perf_counter()
        vecs = vecs.to(self.device, self.store_dtype)
        if vecs.shape[0] > 0:
            a = self.assign(vecs)
            perm, offsets = self.ivf._layout(a)
            vecs, ids, a = vecs[perm].contiguous(), ids[perm], a[perm]
            codes = torch.empty((vecs.shape[0], int(self.token_dim) // 4), dtype=torch.uint8, device=self.device)
            for c0 in range(0, vecs.shape[0], _CHUNK):
                xf = vecs[c0:c0 + _CHUNK].float()
                r = xf - self.ivf.centroids[a[c0:c0 + _CHUNK]]
                codes[c0:c0 + _CHUNK] = pack_codes(encode(r, unit_rows(xf), self.codebook, self.eta))
        else:
            offsets = torch.zeros(self.nlist + 1, dtype=torch.int64, device=self.device)
            codes = torch.empty((0, int(self.token_dim) // 4), dtype=torch.uint8, device=self.device)
        self.rows, self.ids, self.codes, self.list_offsets = vecs.contiguous(), ids.contiguous(), codes, offsets
        self.max_list_len = int((offsets[1:] - offsets[:-1]).max().item())
        torch.cuda.synchronize(self.device)
        self.build_seconds["encoding"] = time.perf_counter() - t0

    # ------------------------------------------------------------------ search
    def _to_device_queries(self, query_vec: numpy.ndarray) -> torch.Tensor:
        if self.rows is None:
            raise _lib.MatchmakerB200Error("search() before index()")
        if query_vec.ndim == 1:
            query_vec = query_vec[numpy.newaxis, :]
        return torch.from_numpy(numpy.ascontiguousarray(query_vec)).to(self.device, dtype=self.store_dtype)

    def search(self, query_vec: numpy.ndarray, top_n: int):
        s, i = self.search_device(self._to_device_queries(query_vec), top_n)
        return s.cpu().numpy(), i.cpu().numpy()

    def coarse(self, q: torch.Tensor):
        """(<q, centroid> [nq, nprobe] f32, leaf ids [nq, nprobe] int64) of the min(100, nlist) best leaves."""
        return interaction.flat_ip_topk(q, self.ivf.c_store, self.nprobe, split_scale=self.ivf.c_scale)

    def luts(self, q: torch.Tensor) -> torch.Tensor:
        """[nq, M, 16] f32: T[m][j] = q[2m] C[m][j][0] + q[2m+1] C[m][j][1]."""
        qv = q.float().view(q.shape[0], -1, 1, 2)
        return (qv[..., 0] * self.codebook[..., 0] + qv[..., 1] * self.codebook[..., 1]).contiguous()

    def shortlist(self, q: torch.Tensor, kr: int):
        """(approximate scores, row positions) [nq, kr] from the code scan of the probed leaves."""
        bias, probes = self.coarse(q)
        return interaction.ah_search(self.luts(q), self.codes, self.list_offsets, probes, bias, kr, self.max_list_len)

    def search_device(self, q: torch.Tensor, top_n: int):
        """Same as search() but device tensors in/out.  No host synchronisation with fp16 storage (fp32 storage reads
        the query scale when the coarse stage splits the queries).  Returns the ids given to index()."""
        rank, world = self._world()
        kr = shortlist_size(self.top_n, top_n)
        q = q.to(self.store_dtype)
        if self.rows.shape[0] > 0:
            _, pos = self.shortlist(q, kr)
            s, i = interaction.ah_reorder(q, self.rows, self.ids, pos, top_n)
        else:
            s = torch.full((q.shape[0], top_n), _NO_RESULT, device=self.device)
            i = torch.full((q.shape[0], top_n), -1, dtype=torch.int64, device=self.device)
        if world > 1:
            s, i = sharding.all_gather_merge(s, i, top_n, self.group)
        return s, i

    def search_unique(self, query_vec: numpy.ndarray, top_n: int, index_hit_top_n: int):
        """The ``maxP->bert_dot`` aggregation, as FlatIPIndexer.search_unique: ``index_hit_top_n`` hits, the ``top_n``
        best distinct ids at their best score."""
        s, i = self.search_device(self._to_device_queries(query_vec), index_hit_top_n)
        s, i = interaction.topk_unique(s, i, top_n)
        return s.cpu().numpy(), i.cpu().numpy()

    # ------------------------------------------------------------------ persistence
    def _shard_file(self, path: str) -> str:
        rank, world = self._world()
        return os.path.join(path, f"rank{rank}of{world}.pt")

    def save(self, path: str):
        """Into the directory `path` (created if missing): one file per rank, `rank<r>of<w>.pt`, with its rows, codes,
        leaf layout, the centroids and the codebook."""
        rank, world = self._world()
        os.makedirs(path, exist_ok=True)
        torch.save({"centroids": self.ivf.centroids.cpu(), "codebook": self.codebook.cpu(), "rows": self.rows.cpu(),
                    "codes": self.codes.cpu(), "ids": self.ids.cpu(), "list_offsets": self.list_offsets.cpu(),
                    "max_list_len": self.max_list_len, "n_total": self.n_total, "lo": getattr(self, "lo", 0),
                    "hi": getattr(self, "hi", self.n_total), "world": world, "rank": rank,
                    "token_dtype": str(self.store_dtype), "nlist": self.nlist, "nprobe": self.nprobe,
                    "top_n": self.top_n, "train_loss": self.train_loss}, self._shard_file(path))

    def load(self, path: str):
        blob = self._load_shard(self._shard_file(path))
        lo, hi = sharding.shard_bounds(blob["n_total"], *self._world())
        self._leaves(int(blob["nlist"]), int(blob["nprobe"]))
        self.ivf.set_centroids(blob["centroids"])
        self.codebook = blob["codebook"].to(self.device)
        self.rows, self.codes = blob["rows"].to(self.device), blob["codes"].to(self.device)
        self.ids, self.list_offsets = blob["ids"].to(self.device), blob["list_offsets"].to(self.device)
        self.max_list_len = int(blob["max_list_len"])
        self.train_loss = list(blob["train_loss"])
        self.n_total, self.lo, self.hi = blob["n_total"], lo, hi
