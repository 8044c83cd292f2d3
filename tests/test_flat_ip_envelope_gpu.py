"""The inner-product top-k across its whole instantiation matrix (tests/flat_ip_cases.py): every compiled instantiation of
the kernel body behind ``flat_ip_topk``, ``ivf_search`` (plain and with ``row_index``) and ``ivf_search_residual``, at
the k, n, nq, dim, cluster, range and merge edges, with every top-k score negative, tie runs longer than a candidate list
straddling rank k, and ids at both ends of the int64 range.

The inputs are integers, so every fp32 sum is exact: scores and ids are held bit-exactly to the fp64 oracle, including
the (-FLT_MAX, -1) tail.  Besides: one row under every cluster size and range count, two runs, a permutation of the
passages with their ids, gather against the plain scan and residual codes against the gather over their decoded rows,
and the plan the library makes on this device."""
import ctypes
import functools

import pytest
import torch

import flat_ip_cases as C
from matchmaker_b200 import _lib, interaction

pytestmark = pytest.mark.gpu
DEV = "cuda"
FLAT_ROWS = [r for r in C.MATRIX if r.mode == "flat"]
IVF_ROWS = [r for r in C.MATRIX if r.mode == "ivf"]
RESIDUAL_ROWS = [r for r in C.MATRIX if r.mode == "residual"]
TORCH = {"f16": torch.float16, "bf16": torch.bfloat16, "e4m3": torch.float8_e4m3fn}


def _dev(x: torch.Tensor, dtype: str) -> torch.Tensor:
    return x.float().to(TORCH[dtype]).to(DEV)


def _take(x: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """x[idx] by rows, through the bytes for e4m3."""
    if x.dtype == torch.float8_e4m3fn:
        return x.view(torch.uint8)[idx].view(torch.float8_e4m3fn)
    return x[idx]


def _env(monkeypatch, cl=None, ranges=None):
    for name, v in (("MMB200_FLATIP_CLUSTER", cl), ("MMB200_FLATIP_RANGES", ranges)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))


def _exact(got, ref, what):
    gs, gi = (t.cpu() for t in got)
    rs, ri = ref
    assert gs.shape == rs.shape and gi.shape == ri.shape, f"{what}: shape {tuple(gs.shape)} vs {tuple(rs.shape)}"
    bad = (gs != rs) | (gi != ri)
    assert not bad.any(), (f"{what}: {int(bad.sum())}/{bad.numel()} differ, first at {bad.nonzero()[0].tolist()}: "
                           f"({gs[bad][0].item()}, {gi[bad][0].item()}) vs ({rs[bad][0].item()}, {ri[bad][0].item()})")


@functools.lru_cache(maxsize=4)
def _flat_inputs(row: C.Row):
    """(queries, passages, split scale) on the device as flat_ip_topk takes them."""
    c = C.make_case(row)
    if row.dtype == "split":
        ps, scale = interaction.flat_ip_split_f32(c.p.float().to(DEV), "passages")
        return c.q.float().to(DEV), ps, scale
    return _dev(c.q, row.dtype), _dev(c.p, row.dtype), None


def _flat(row: C.Row, q, p, scale, ids=None):
    return interaction.flat_ip_topk(q, p, row.k, ids=ids, id_base=row.id_base, split_scale=scale)


@pytest.mark.parametrize("row", FLAT_ROWS, ids=str)
def test_flat_rows_bit_exact(row, monkeypatch):
    """flat_ip_topk under the row's plan overrides; a second run and a permutation of the passages with their ids give
    the same bits."""
    _env(monkeypatch, row.cl, row.ranges)
    c = C.make_case(row)
    q, p, scale = _flat_inputs(row)
    ids = None if c.ids is None else c.ids.to(DEV)
    ref = C.expected(row)
    got = _flat(row, q, p, scale, ids)
    _exact(got, ref, str(row))
    again = _flat(row, q, p, scale, ids)
    assert torch.equal(again[0], got[0]) and torch.equal(again[1], got[1]), "two runs differ"
    perm = torch.randperm(row.n, generator=torch.Generator().manual_seed(row.seed)).to(DEV)
    pid = C.row_ids(row, c).to(DEV)[perm]
    _exact(interaction.flat_ip_topk(q, _take(p, perm), row.k, ids=pid, split_scale=scale), ref, f"{row} permuted")


def test_one_row_under_every_cluster_size_and_range_count(monkeypatch):
    row = C.METAMORPHIC_ROW
    c = C.make_case(row)
    q, p, scale = _flat_inputs(row)
    ref = C.expected(row)
    first = None
    for cl in (1, 2, 4):
        for ranges in (1, None, 32):
            _env(monkeypatch, cl, ranges)
            got = _flat(row, q, p, scale, c.ids.to(DEV))
            _exact(got, ref, f"{row} CL {cl} ranges {ranges or 'auto'}")
            first = first or got
            assert torch.equal(got[0], first[0]) and torch.equal(got[1], first[1])


def test_plan_on_the_device(monkeypatch):
    """mmb200_flat_ip_plan at this device's SM count gives every flat row the cluster size it claims and the range
    count of the restatement."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    lib = _lib.load()
    for row in FLAT_ROWS:
        _env(monkeypatch, row.cl, row.ranges)
        out = (ctypes.c_int32 * 8)()
        assert lib.mmb200_flat_ip_plan(row.nq, row.n, row.k, sm, out) == _lib.OK, _lib.last_error()
        (claimed,) = C.dispatched(row)
        assert claimed == C.flat_inst(row.dtype, out[5], C.epl_for_k(row.k)), str(row)
        assert out[2] == row.plan(sm)["n_ranges"], str(row)


def _ivf_args(row: C.Row, c: C.Case):
    return (_dev(c.q, row.dtype), c.offsets.to(DEV), c.probes.to(DEV))


@pytest.mark.parametrize("row", IVF_ROWS, ids=str)
def test_ivf_rows_bit_exact(row, monkeypatch):
    """ivf_search over the rows in list order, and with row_index over the shuffled store with padding rows: both equal
    the oracle over the union of each query's probed lists, and each other.  e4m3: the plain scan is refused; the
    gather gives the same bits with its queries cut into batches by a lowered workspace cap, and at full probe it gives
    the bits of the e4m3 flat scan."""
    c = C.make_case(row)
    q, offsets, probes = _ivf_args(row, c)
    ref = C.expected(row)
    rows = _dev(c.p, row.dtype)
    args = (c.store_ids.to(DEV), offsets, probes, row.k, row.max_list_len)
    gather = interaction.ivf_search(q, _dev(c.store, row.dtype), *args, row_index=c.row_index.to(DEV))
    _exact(gather, ref, f"{row} gather")
    if row.dtype == "e4m3":
        with pytest.raises(_lib.MatchmakerB200Error):
            interaction.ivf_search(q, rows, c.ids.to(DEV), offsets, probes, row.k, row.max_list_len)
        lib = _lib.load()
        nprobe, nlist = probes.shape[1], len(row.lists)
        def wsb(b):
            return lib.mmb200_ivf_workspace_bytes(b, nprobe, nlist, row.max_list_len, row.dim, row.k, _lib.F8E4M3)
        monkeypatch.setattr(interaction, "IVF_WORKSPACE_CAP", wsb(max(1, row.nq // 3)))
        assert interaction.ivf_query_batch(row.nq, wsb, interaction.IVF_WORKSPACE_CAP) < row.nq
        batched = interaction.ivf_search(q, _dev(c.store, row.dtype), *args, row_index=c.row_index.to(DEV))
        assert torch.equal(batched[0], gather[0]) and torch.equal(batched[1], gather[1]), "batched queries differ"
        monkeypatch.undo()
        if nlist > interaction.IVF_MAX_PROBE:
            return
        full = torch.arange(nlist).repeat(row.nq, 1).to(DEV)
        s_g, i_g = interaction.ivf_search(q, _dev(c.store, row.dtype), c.store_ids.to(DEV), offsets, full, row.k,
                                          row.max_list_len, row_index=c.row_index.to(DEV))
        s_f, i_f = interaction.flat_ip_topk(q, rows, row.k, ids=c.ids.to(DEV))
        assert torch.equal(s_g, s_f) and torch.equal(i_g, i_f), "full probe differs from the flat scan"
        return
    plain = interaction.ivf_search(q, rows, c.ids.to(DEV), offsets, probes, row.k, row.max_list_len)
    _exact(plain, ref, f"{row} plain")
    assert torch.equal(gather[0], plain[0]) and torch.equal(gather[1], plain[1])


@pytest.mark.parametrize("row", RESIDUAL_ROWS, ids=str)
def test_residual_rows_bit_exact(row):
    """ivf_search_residual over codes with integer tables equals the oracle over the decoded rows, and the gather scan
    over those rows."""
    c = C.make_case(row)
    q, offsets, probes = _ivf_args(row, c)
    ref = C.expected(row)
    ids, row_index = c.store_ids.to(DEV), c.row_index.to(DEV)
    got = interaction.ivf_search_residual(q, torch.from_numpy(c.codes).to(DEV), torch.from_numpy(c.base).to(DEV),
                                          torch.from_numpy(c.weight).to(DEV), row.bits, ids, row_index, offsets, probes,
                                          row.k, row.max_list_len)
    _exact(got, ref, f"{row} residual")
    gather = interaction.ivf_search(q, c.store.half().to(DEV), ids, offsets, probes, row.k, row.max_list_len,
                                    row_index=row_index)
    assert torch.equal(gather[0], got[0]) and torch.equal(gather[1], got[1])


def test_empty_query_batch():
    p = torch.ones(300, 64, dtype=torch.float16, device=DEV)
    s, i = interaction.flat_ip_topk(p[:0], p, 10)
    assert s.shape == (0, 10) and i.shape == (0, 10) and s.dtype == torch.float32 and i.dtype == torch.int64
