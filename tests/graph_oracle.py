"""CPU restatement of the graph index, in fp64 and integer logic: the k-NN graph with its tie-break, the rank-based
detour counts and pruning, the reverse-edge merge, the entry sample and the beam search with an exact visited set.
With integer-valued vectors every score is exact, so the GPU must agree with it bit for bit."""
import numpy as np
import torch

NO_RESULT = -3.4028234663852886e38
SEED = 1234


def _ranked(scores: np.ndarray, pos: np.ndarray) -> np.ndarray:
    """pos ordered by (score desc, pos asc)."""
    return pos[np.lexsort((pos, -scores))]


def knn(x: torch.Tensor, K: int) -> np.ndarray:
    """[n, K] int32: each row's K best other rows under (score desc, position asc), -1 where there are fewer."""
    x64 = x.double().numpy()
    n = x64.shape[0]
    s = x64 @ x64.T
    out = np.full((n, K), -1, dtype=np.int32)
    for u in range(n):
        others = np.delete(np.arange(n), u)
        r = _ranked(s[u, others], others)[:K]
        out[u, :len(r)] = r
    return out


def detour_counts(knn_lists: np.ndarray) -> np.ndarray:
    """[n, K]: edge u -> v = N(u)[j] has a detour through w = N(u)[i] for every i < j with v = N(w)[p], p < j."""
    n, K = knn_lists.shape
    out = np.zeros((n, K), dtype=np.int64)
    idx = np.arange(K)
    for u in range(n):
        nu = knn_lists[u]
        rank = np.full(n + 1, -1, dtype=np.int64)     # rank[v] = j of v in N(u); index n catches the -1 entries
        valid = nu >= 0
        rank[nu[valid][::-1]] = idx[valid][::-1]       # a repeated id keeps its first rank
        w = np.where(valid, nu, 0)
        nw = knn_lists[w]                              # [K (i), K (p)]
        J = rank[np.where(nw >= 0, nw, n)]
        ok = valid[:, None] & (J > idx[:, None]) & (J > idx[None, :])
        out[u] = np.bincount(J[ok], minlength=K)[:K]
    return out


def prune(knn_lists: np.ndarray, R: int, counts: np.ndarray = None) -> np.ndarray:
    """[n, R] int32: the R valid edges with the fewest detours (ties by rank), in rank order, -1 padded."""
    if counts is None:
        counts = detour_counts(knn_lists)
    n, K = knn_lists.shape
    out = np.full((n, R), -1, dtype=np.int32)
    for u in range(n):
        js = [j for j in range(K) if knn_lists[u, j] >= 0]
        keep = sorted(sorted(js, key=lambda j: (counts[u, j], j))[:R])
        out[u, :len(keep)] = knn_lists[u, keep]
    return out


def reverse_merge(pruned: np.ndarray) -> np.ndarray:
    """[n, R] int32: head ceil(R/2) of u's pruned list, then the w with u in the head of w's list ordered by (that rank,
    w), then the rest of u's list; duplicates skipped, cut at R, -1 padded."""
    n, R = pruned.shape
    H = (R + 1) // 2
    rev = [[] for _ in range(n)]
    for w in range(n):
        for r in range(H):
            v = int(pruned[w, r])
            if v >= 0:
                rev[v].append((r, w))
    out = np.full((n, R), -1, dtype=np.int32)
    for u in range(n):
        seq = [int(v) for v in pruned[u, :H] if v >= 0] + [w for _, w in sorted(rev[u])] + \
              [int(v) for v in pruned[u, H:] if v >= 0]
        lst = []
        for v in seq:
            if v not in lst:
                lst.append(v)
            if len(lst) == R:
                break
        out[u, :len(lst)] = lst
    return out


def build(x: torch.Tensor, R: int, K: int) -> np.ndarray:
    return reverse_merge(prune(knn(x, K), R))


def entry_positions(n: int) -> np.ndarray:
    e = min(n, max(1024, n // 128))
    return np.random.RandomState(SEED).permutation(n)[:e].astype(np.int64)


def search(q: torch.Tensor, x: torch.Tensor, graph: np.ndarray, entries: np.ndarray, L: int, k: int, ids=None):
    """Beam search of every query: (scores [nq, k] f32, ids [nq, k] int64, distinct rows visited [nq]).

    The starting list is the min(L, E) best entry rows; each step expands the best list entry not yet expanded, scores
    its unvisited neighbours and keeps the L best under (score desc, position asc); it stops when every entry has been
    expanded or after 2 * L steps."""
    x64, q64 = x.double().numpy(), q.double().numpy()
    ids = np.arange(x64.shape[0]) if ids is None else np.asarray(ids)
    nq = q64.shape[0]
    out_s = np.full((nq, k), NO_RESULT, dtype=np.float32)
    out_i = np.full((nq, k), -1, dtype=np.int64)
    visited_n = np.zeros(nq, dtype=np.int64)
    for a in range(nq):
        es = x64[entries] @ q64[a]
        start = _ranked(es, entries)[:min(L, len(entries))]
        score = {int(p): float(x64[p] @ q64[a]) for p in start}
        visited = set(score)
        lst = sorted(visited, key=lambda p: (-score[p], p))[:L]
        parents = set()
        for _ in range(2 * L):
            cand = [p for p in lst if p not in parents]
            if not cand:
                break
            node = cand[0]
            parents.add(node)
            new = [int(v) for v in graph[node] if v >= 0 and int(v) not in visited]
            for v in new:
                visited.add(v)
                score[v] = float(x64[v] @ q64[a])
            if new:
                lst = sorted(lst + new, key=lambda p: (-score[p], p))[:L]
        top = lst[:k]
        out_s[a, :len(top)] = [score[p] for p in top]
        out_i[a, :len(top)] = ids[top]
        visited_n[a] = len(visited)
    return torch.from_numpy(out_s), torch.from_numpy(out_i), visited_n


def integer_rows(n: int, dim: int, seed: int, dup: int = 0, lim: int = 8) -> torch.Tensor:
    """[n, dim] integer-valued fp32 rows in [-lim, lim] (exact in fp16, every dot product exact in fp32); the last
    `dup` rows copy earlier rows."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-lim, lim + 1, (n, dim), generator=g).float()
    if dup:
        src = torch.randint(0, n - dup, (dup,), generator=g)
        x[n - dup:] = x[src]
    return x
