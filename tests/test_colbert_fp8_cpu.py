"""The E4M3 token store without a GPU: the scale rule and quantizer against the oracle, the oracle against a
hand-worked case, the indexers' configuration envelope, the C ABI's constant and envelope, the all-reduced store
scale on a world-size-2 gloo group, and the compiled e4m3 kernels (QGMMA, TMA, mbarrier waits, uniform issue)."""
import math
import os
import re
import shutil
import socket
import subprocess

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import colbert_fp8_oracle as F
from matchmaker_b200 import _lib, build, interaction
from matchmaker_b200.retrieval import colbert_e2e


# ----------------------------------------------------------------------------------------------------------------------
# scale rule and quantizer
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("amax", [448.0, 449.0, 224.0, 896.0, 1.0, 0.875, 0.8750001, 0.5, 2.0 ** -20, 3.0 * 2.0 ** 7,
                                  65504.0, 2.0 ** -24, 1e-30, 1e-40, 3.0e38, 0.0])
def test_scale_rule_is_the_largest_power_of_two_that_fits(amax):
    a32 = float(torch.tensor(amax, dtype=torch.float32))
    s = interaction.fp8_store_scale(a32)
    assert s == F.scale_log2(a32)
    if a32 > 0:
        assert math.ldexp(a32, s) <= 448.0 < math.ldexp(a32, s + 1)
    else:
        assert s == 0
    dev = interaction.fp8_scale_log2(torch.tensor([a32, 0.0, a32], dtype=torch.float32))
    assert dev.dtype == torch.int32 and dev.tolist() == [s, 0, s]


def test_scale_rule_at_powers_of_two():
    for e in range(-60, 60):
        assert interaction.fp8_store_scale(2.0 ** e) == 8 - e      # 2^e * 2^(8-e) = 256 <= 448 < 512
        assert interaction.fp8_store_scale(448.0 * 2.0 ** e) == -e


@pytest.mark.parametrize("bad", [math.inf, -math.inf, math.nan])
def test_non_finite_store_maximum_raises(bad):
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.fp8_store_scale(bad)
    with pytest.raises(ValueError):
        F.scale_log2(bad)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_quantize_is_the_cast_of_the_scaled_value(dtype):
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(7, 9, 128, generator=g) * torch.logspace(-6, 3, 7)[:, None, None]).to(dtype)
    x[3] = 0
    s = interaction.fp8_scale_log2(x.abs().amax(dim=(1, 2)))
    got = interaction.fp8_quantize(x, s)
    ref, rs = F.quantize_queries(x)
    assert s.tolist() == rs.tolist()
    assert got.dtype == torch.float8_e4m3fn
    assert torch.equal(got.view(torch.uint8), ref.view(torch.uint8))
    assert float(got.float().abs().max()) <= 448.0
    one = interaction.fp8_quantize(x[1], int(s[1]))
    assert torch.equal(one.view(torch.uint8), F.quantize(x[1], int(s[1])).view(torch.uint8))


def test_unscale_is_exact_and_keeps_void_scores():
    s = torch.tensor([[3.0, -1.5, -3.4028234663852886e38], [1.0, float("-inf"), 7.0]])
    out = interaction.fp8_unscale(s, torch.tensor([2, -3]))
    assert out[0].tolist() == [0.75, -0.375, -3.4028234663852886e38]
    assert out[1].tolist() == [8.0, float("-inf"), 56.0]


def test_oracle_on_a_hand_worked_case():
    """Two query tokens against a store of three rows in two passages, worked by hand.

    q = [[1, 2], [0.5, -1]] -> max |q| = 2, s_q = 7 (2 * 2^7 = 256 <= 448 < 512): stored [[128, 256], [64, -128]].
    rows = [[3, 0], [1, 1], [-2, 4]] -> max 4, s_d = 6 (256 <= 448): stored [[192, 0], [64, 64], [-128, 256]].
    Scaled token scores: token 0 = [24576, 24576, 49152], token 1 = [12288, -4096, -40960].
    Passage 0 (rows 0, 1): 24576 + 12288 = 36864; passage 1 (row 2): 49152 - 40960 = 8192.
    Unscaled by 2^-13: 4.5 and 1.0, the fp64 max-sim of the original values (all of them exact in e4m3)."""
    q = torch.tensor([[[1.0, 2.0], [0.5, -1.0]]])
    rows = torch.tensor([[3.0, 0.0], [1.0, 1.0], [-2.0, 4.0]])
    q8, sq = F.quantize_queries(q)
    sd = F.scale_log2(4.0)
    assert sq.tolist() == [7] and sd == 6
    r8 = F.quantize(rows, sd)
    assert q8.float().tolist() == [[[128.0, 256.0], [64.0, -128.0]]]
    assert r8.float().tolist() == [[192.0, 0.0], [64.0, 64.0], [-128.0, 256.0]]
    sc, tol = F.maxsim_store(q8, r8, [0, 2, 3], 8, c=0.0)
    assert sc.tolist() == [[36864.0, 8192.0]]
    assert (sc * 2.0 ** -(7 + 6)).tolist() == [[4.5, 1.0]]
    sc1, _ = F.maxsim_store(q8, r8, [0, 2, 3], 1, c=0.0)   # max_doc_len 1: passage 0 reads row 0 only
    assert sc1.tolist() == [[36864.0, 8192.0]]
    assert tol[0, 0] == 2.0 ** -22 * (24576 + 12288)


# ----------------------------------------------------------------------------------------------------------------------
# configuration
# ----------------------------------------------------------------------------------------------------------------------
def _cfg(**kw):
    c = {"token_dim": 128, "faiss_use_gpu": True, "token_dtype": "float16", "faiss_ivf_list_count": 8,
         "faiss_ivf_search_probe_count": 2, "colbert_store_dtype": "float8_e4m3"}
    c.update(kw)
    return c


def test_indexers_accept_the_fp8_store():
    from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer
    for cls in (ColBERTEndToEndIndexer, ColBERTIVFIndexer):
        for dim in (128, 256, 768, 1024):
            assert cls(_cfg(token_dim=dim), device=torch.device("cpu")).fp8
        plain = dict(_cfg())
        del plain["colbert_store_dtype"]
        assert not cls(plain, device=torch.device("cpu")).fp8


@pytest.mark.parametrize("bad", [{"colbert_store_dtype": "float8_e5m2"}, {"colbert_store_dtype": "float16"},
                                 {"token_dim": 64}, {"token_dim": 192}, {"token_dim": 1152},
                                 {"colbert_residual_bits": 2}])
def test_indexers_reject_configurations_outside_the_envelope(bad):
    from matchmaker_b200.retrieval import ColBERTEndToEndIndexer, ColBERTIVFIndexer, ColBERTResidualIndexer
    for cls in (ColBERTEndToEndIndexer, ColBERTIVFIndexer, ColBERTResidualIndexer):
        cfg = _cfg(**bad)
        if cls is ColBERTResidualIndexer:
            cfg.setdefault("colbert_residual_bits", 2)
        with pytest.raises(_lib.MatchmakerB200Error):
            cls(cfg, device=torch.device("cpu"))


# ----------------------------------------------------------------------------------------------------------------------
# C ABI
# ----------------------------------------------------------------------------------------------------------------------
def test_header_defines_the_e4m3_dtype():
    hdr = open(os.path.join(build.INCLUDE, "matchmaker_b200.h")).read()
    assert re.search(r"#define MMB200_F8E4M3 4\b", hdr)
    assert _lib.F8E4M3 == 4


@pytest.mark.parametrize("dim", [64, 192, 1152])
def test_entry_points_reject_e4m3_outside_the_envelope(dim):
    """Checked before any device is touched: the arguments are never dereferenced."""
    lib = _lib.load()
    p = 1 << 12   # a 16-byte aligned stand-in pointer
    rc = lib.mmb200_flat_ip_topk(p, p, None, p, p, p, 1 << 30, 1, 1000, dim, 10, _lib.F8E4M3, 0, None)
    assert rc == _lib.ERR_INVALID
    rc = lib.mmb200_maxsim_store_fwd(p, p, p, p, p, p, 1, 100, 10, 1, 32, 16, dim, _lib.F8E4M3, _lib.IMPL_AUTO, None)
    assert rc == _lib.ERR_INVALID
    assert lib.mmb200_ivf_workspace_bytes(4, 2, 8, 100, dim, 10, _lib.F8E4M3) == 0
    rc = lib.mmb200_ivf_search_gather(p, p, p, p, p, p, p, p, p, 1 << 30, 4, 2, 8, 100, 100, dim, 10, _lib.F8E4M3, None)
    assert rc == _lib.ERR_INVALID


def test_e4m3_entry_points_refuse_other_kernels():
    lib = _lib.load()
    p = 1 << 12
    for impl in (_lib.IMPL_SIMT, _lib.IMPL_TCGEN05):
        rc = lib.mmb200_maxsim_store_fwd(p, p, p, p, p, p, 1, 100, 10, 1, 32, 16, 128, _lib.F8E4M3, impl, None)
        assert rc == _lib.ERR_UNSUPPORTED
    # e4m3 rows are scanned in gather mode only, and never as residual codes
    rc = lib.mmb200_ivf_search(p, p, p, p, p, p, p, p, 1 << 30, 4, 2, 8, 100, 100, 128, 10, _lib.F8E4M3, None)
    assert rc == _lib.ERR_INVALID
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.maxsim_store(torch.zeros(1, 4, 128, dtype=torch.float8_e4m3fn), torch.zeros(4, 128),
                                 torch.tensor([0, 4]), torch.zeros(1), torch.zeros(1), 4)


# ----------------------------------------------------------------------------------------------------------------------
# the store scale over ranks
# ----------------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _scale_worker(rank, world, port, maxima, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        s = colbert_e2e.fp8_store_scale(torch.tensor(maxima[rank], dtype=torch.float32))
        torch.save(s, os.path.join(out_dir, f"r{rank}.pt"))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(120)
@pytest.mark.parametrize("maxima", [(3.0, 0.25), (0.0, 700.0), (0.0, 0.0)])
def test_gloo_world2_store_scale_is_the_scale_of_the_global_maximum(tmp_path, maxima):
    mp.spawn(_scale_worker, args=(2, _free_port(), maxima, str(tmp_path)), nprocs=2, join=True)
    got = [torch.load(os.path.join(tmp_path, f"r{r}.pt")) for r in range(2)]
    assert got[0] == got[1] == F.scale_log2(max(maxima))
    assert colbert_e2e.fp8_store_scale(torch.tensor(max(maxima))) == got[0]   # no process group: the local maximum


# ----------------------------------------------------------------------------------------------------------------------
# compiled kernels
# ----------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sass():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        out = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
    except (FileNotFoundError, subprocess.TimeoutExpired) as e:
        pytest.skip(f"cuobjdump unavailable: {e}")
    if out.returncode != 0:
        pytest.skip("cuobjdump failed: " + out.stderr[-200:])
    funcs, name = {}, None
    for line in out.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name is not None:
            funcs[name].append(line)
    return {k: "\n".join(v) for k, v in funcs.items()}


def _mma_lines(text, op):
    return [l for l in text.splitlines() if op in l and "gdesc[URZ]" not in l]


@pytest.mark.parametrize("needle,count", [("flat_ip_tc_fp8_kernel", 6), ("flat_ip_tc_gather_fp8_kernel", 2),
                                          ("maxsim_tc_fp8_kernel", 8)])
def test_fp8_kernels_are_e4m3_wgmma_kernels_fed_by_tma(sass, needle, count):
    ks = {k: v for k, v in sass.items() if needle in k}
    assert len(ks) == count, list(ks)
    for name, text in ks.items():
        q = _mma_lines(text, "QGMMA")
        assert q and all(".E4M3.E4M3" in l for l in q), f"{name}: no e4m3 wgmma (QGMMA .E4M3)"
        assert not _mma_lines(text, "HGMMA"), f"{name}: a 16-bit wgmma in an e4m3 kernel"
        assert "UTMALDG" in text, f"{name}: no TMA tensor load (UTMALDG)"
        assert "SYNCS.PHASECHK" in text, f"{name}: no mbarrier wait"
        lines = [l for l in text.splitlines() if re.search(r"/\*[0-9a-f]{4}\*/", l)]
        for i, l in enumerate(lines):
            if "UTMALDG" in l or ("QGMMA" in l and "gdesc[URZ]" not in l):
                assert "BRA.U.ANY" not in " ".join(lines[i + 1:i + 3]), f"{name}: MMA or TMA issue inside a waterfall loop"


def test_fp8_flat_ip_cluster_instantiations_multicast(sass):
    ks = {k: v for k, v in sass.items() if "flat_ip_tc_fp8_kernel" in k}
    assert any(".MULTICAST" in v.upper() for v in ks.values())
