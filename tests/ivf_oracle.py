"""CPU restatement of the IVF index: the search is the exact top-k over the union of each query's probed lists (checked
with oracle.flat_ip_search / flat_ip_check_exact on the union's rows), and one spherical k-means iteration in fp64."""
import torch

from oracle import interaction_oracle as O

NO_RESULT = -3.4028234663852886e38


def union_rows(list_offsets: torch.Tensor, probes_row: torch.Tensor) -> torch.Tensor:
    """Row indices of the probed lists of one query (ids outside [0, nlist) probe nothing)."""
    nlist = list_offsets.numel() - 1
    parts = [torch.arange(int(list_offsets[l]), int(list_offsets[l + 1])) for l in probes_row.tolist() if 0 <= l < nlist]
    return torch.cat(parts) if parts else torch.zeros(0, dtype=torch.int64)


def ivf_search(queries, rows, ids, list_offsets, probes, k):
    """(scores [nq, k] f32, ids [nq, k] i64): flat_ip_search of every query over its union, (-FLT_MAX, -1) tail."""
    out_s = torch.full((queries.shape[0], k), NO_RESULT)
    out_i = torch.full((queries.shape[0], k), -1, dtype=torch.int64)
    for r in range(queries.shape[0]):
        u = union_rows(list_offsets, probes[r])
        if u.numel():
            s, i = O.flat_ip_search(queries[r:r + 1].float(), rows[u], ids[u], k)
            out_s[r], out_i[r] = s[0], i[0]
    return out_s, out_i


def ivf_check_exact(queries, rows, ids, list_offsets, probes, got_s, got_i, k) -> dict:
    """flat_ip_check_exact per query on the union's rows, plus the (-FLT_MAX, -1) tail past the union's size."""
    got_s, got_i = got_s.cpu(), got_i.cpu()
    tot = {"decided": 0, "undecided": 0}
    for r in range(queries.shape[0]):
        u = union_rows(list_offsets, probes[r])
        n = u.numel()
        if n:
            st = O.flat_ip_check_exact(queries[r:r + 1], rows[u], ids[u], got_s[r:r + 1], got_i[r:r + 1], k)
            tot["decided"] += st["decided"]
            tot["undecided"] += st["undecided"]
        assert torch.all(got_i[r, n:] == -1) and torch.all(got_s[r, n:] == NO_RESULT), f"query {r}: tail past {n} rows"
    return tot


def kmeans_step(x: torch.Tensor, c: torch.Tensor):
    """One spherical k-means iteration in fp64 from centroids c (as the device sees them): (assignment [n] = argmax
    inner product, lowest list on ties; new unit centroids [nlist, dim], zero rows for empty lists; gap [n] between the
    best and second-best inner product, to tell near-ties)."""
    x64, c64 = x.double(), c.double()
    s = x64 @ c64.T
    top2 = torch.topk(s, min(2, c.shape[0]), dim=1)
    assign = torch.argmax(s, dim=1)
    gap = (top2.values[:, 0] - top2.values[:, -1]) if c.shape[0] > 1 else torch.full((x.shape[0],), float("inf"))
    sums = torch.zeros_like(c64).index_add_(0, assign, x64)
    norm = sums.norm(dim=1, keepdim=True)
    return assign, torch.where(norm > 0, sums / norm.clamp_min(1e-300), torch.zeros_like(sums)), gap


def ivf_check_split(queries, rows, ids, list_offsets, probes, got_s, got_i, k) -> dict:
    """Checker for fp32 storage (the fp16 hi / lo split, 22 mantissa bits per operand), as the flat-IP fp32 tests check
    it: per query over the union's rows, scores within 1e-5 relative of fp64 and ids equal to the fp64 ranking wherever
    neighbouring fp64 scores differ by more than 2e-5 relative; the (-FLT_MAX, -1) tail past the union's size."""
    got_s, got_i = got_s.cpu().double(), got_i.cpu()
    tot = {"decided": 0, "undecided": 0}
    for r in range(queries.shape[0]):
        u = union_rows(list_offsets, probes[r])
        n = u.numel()
        kk = min(k, n)
        if kk:
            s64 = rows[u].double() @ queries[r].double()
            ref_s, pos = torch.topk(s64, kk)
            ref_i = ids[u][pos]
            assert ((got_s[r, :kk] - ref_s).abs() <= 1e-5 * ref_s.abs().clamp(min=1.0)).all(), f"query {r}: scores"
            tol = 2e-5 * ref_s.abs().clamp(min=1.0)
            decided = torch.ones(kk, dtype=torch.bool)
            if kk > 1:
                gaps = ref_s[:-1] - ref_s[1:]
                decided[1:] &= gaps > tol[1:]
                decided[:-1] &= gaps > tol[:-1]
            if kk < n:   # the last rank is also compared against the first row left out
                decided[-1] &= bool(ref_s[-1] - torch.topk(s64, kk + 1).values[-1] > tol[-1])
            assert torch.equal(got_i[r, :kk][decided], ref_i[decided]), f"query {r}: ids"
            tot["decided"] += int(decided.sum())
            tot["undecided"] += int((~decided).sum())
        assert torch.all(got_i[r, n:] == -1) and torch.all(got_s[r, n:] == NO_RESULT), f"query {r}: tail past {n} rows"
    return tot
