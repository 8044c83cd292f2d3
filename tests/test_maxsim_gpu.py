"""Parity of the CUDA max-sim path (through the C ABI) with the oracle / golden vectors.
Bar: <= 1e-3 relative fp32 (BASELINE.json north_star); fp16/bf16 inputs are upcast for the oracle so
products are exact and only accumulation order differs."""
import pytest
import torch

from conftest import assert_close_rel, load_golden
from matchmaker_b200 import _lib, interaction
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _cuda(*ts):
    return [None if t is None else t.to(DEV) for t in ts]


def test_golden_small_fp32_masked_agg_allpairs():
    g = load_golden("colbert_small")
    q, d, qm, dm = _cuda(g["q"], g["d"], g["q_mask"], g["d_mask"])
    assert_close_rel(interaction.maxsim(q, d, qm, dm), g["score"], what="forward")
    assert_close_rel(interaction.maxsim(q, d), g["agg"], what="forward_aggregation")
    # colbert.py:158 indexes the document mask by the query position; reproduced on request
    assert_close_rel(interaction.maxsim_allpairs(q, qm, d, dm, reference_mask_indexing=True), g["allpairs"],
                     what="inbatch (reference mask indexing)")
    own = O.maxsim_allpairs_own_masks(g["q"], g["q_mask"], g["d"], g["d_mask"])
    assert_close_rel(interaction.maxsim_allpairs(q, qm, d, dm), own, what="inbatch (own masks)")


@pytest.mark.parametrize("impl", ["tcgen05", "tcgen05_docm", "simt", "auto"])
def test_golden_cfg3_shape_fp16(impl):
    g = load_golden("colbert_cfg3")
    q, d, qm, dm = _cuda(g["q"], g["d"], g["q_mask"], g["d_mask"])
    s = interaction.maxsim(q, d, qm, dm, docs_per_query=int(g["docs_per_query"]), impl=impl)
    assert_close_rel(s, g["score"], what=f"cfg3 {impl}")


SHAPES = [  # n_q, docs_per_query, Lq, Ld, dim, dtype
    (5, 3, 32, 180, 128, torch.float16),
    (3, 7, 17, 300, 64, torch.float16),     # KBS=1, 3 tiles, ragged Lq
    (4, 2, 64, 57, 256, torch.bfloat16),    # NPAD=64, single tile
    (2, 5, 128, 129, 192, torch.float16),   # NPAD=128 (four wgmma N = 32 chunks), odd k-block count
    (300, 1, 32, 180, 128, torch.float16),  # query changes every pair; more pairs than SMs
    (1, 1, 1, 1, 64, torch.float16),
    (2, 4, 32, 255, 128, torch.bfloat16),   # Ld + 1 == 256: one 256-row tile in the queries-on-M kernel
    (2, 4, 32, 256, 128, torch.float16),    # Ld + 1 == 257: two tiles
    (2, 3, 30, 700, 64, torch.float16),     # long documents, three tiles
]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("impl", ["tcgen05", "tcgen05_docm", "simt"])
def test_seeded_vs_oracle(shape, impl):
    n_q, dpq, Lq, Ld, dim, dt = shape
    q, d, qm, dm = O.synth_colbert_inputs(n_q, dpq, Lq, Ld, dim, seed=99 + Lq + Ld, dtype=dt, full_q=False)
    ref = O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, dpq)
    cq, cd, cqm, cdm = _cuda(q, d, qm, dm)
    got = interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=dpq, impl=impl)
    assert_close_rel(got, ref, what=f"{shape} {impl}")
    # unmasked aggregation (colbert.py:100-112)
    ref2 = O.maxsim_one_query_many_docs(q.float(), d.float(), None, None, dpq)
    assert_close_rel(interaction.maxsim(cq, cd, docs_per_query=dpq, impl=impl), ref2, what=f"{shape} {impl} nomask")


@pytest.mark.parametrize("mdt", [torch.bool, torch.uint8, torch.int32, torch.int64, torch.float32, torch.float16])
def test_mask_dtypes(mdt):
    q, d, qm, dm = O.synth_colbert_inputs(3, 4, 32, 100, 128, seed=7, full_q=False)
    ref = O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, 4)
    cq, cd = _cuda(q, d)
    got = interaction.maxsim(cq, cd, qm.to(DEV).to(mdt), dm.to(DEV).to(mdt), docs_per_query=4)
    assert_close_rel(got, ref, what=str(mdt))


def test_fully_masked_doc_and_query_token_edge_cases():
    q, d, qm, dm = O.synth_colbert_inputs(2, 3, 32, 180, 128, seed=11)
    dm[3] = 0          # document with no real token: every position scores -1000
    dm[4, 1:] = 0      # single-token document
    qm[1, 5:] = 0
    qm[0] = 0          # query with no real token: score 0
    ref = O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, 3)
    cq, cd, cqm, cdm = _cuda(q, d, qm, dm)
    for impl in ("tcgen05", "tcgen05_docm", "simt"):
        assert_close_rel(interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=3, impl=impl), ref, what=impl)
    assert ref[3].item() == -1000.0 * 5


def test_non_prefix_masks():
    q, d, qm, dm = O.synth_colbert_inputs(2, 2, 32, 180, 128, seed=12)
    g = torch.Generator().manual_seed(3)
    dm = (torch.rand(dm.shape, generator=g) > 0.4).long()
    qm = (torch.rand(qm.shape, generator=g) > 0.3).long()
    ref = O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, 2)
    cq, cd, cqm, cdm = _cuda(q, d, qm, dm)
    for impl in ("tcgen05", "tcgen05_docm", "simt"):
        assert_close_rel(interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=2, impl=impl), ref, what=impl)


def test_pair_index_arrays_and_allpairs_fp16():
    q, d, qm, dm = O.synth_colbert_inputs(6, 1, 32, 90, 128, seed=13, full_q=False)
    ref_quirk = O.maxsim_allpairs(q.float(), qm, d.float(), dm)
    ref = O.maxsim_allpairs_own_masks(q.float(), qm, d.float(), dm)
    cq, cd, cqm, cdm = _cuda(q, d, qm, dm)
    for impl in ("tcgen05", "tcgen05_docm", "simt"):
        assert_close_rel(interaction.maxsim_allpairs(cq, cqm, cd, cdm, impl=impl), ref, what=f"allpairs {impl}")
        assert_close_rel(interaction.maxsim_allpairs(cq, cqm, cd, cdm, impl=impl, reference_mask_indexing=True),
                         ref_quirk, what=f"allpairs quirk {impl}")
    pq = torch.tensor([5, 0, 0, 3, 3, 3, 1], dtype=torch.int32, device=DEV)
    pd = torch.tensor([0, 5, 2, 2, 4, 1, 1], dtype=torch.int32, device=DEV)
    got = interaction.maxsim(cq, cd, cqm, cdm, pair_q=pq, pair_d=pd)
    assert_close_rel(got, ref[pq.long().cpu(), pd.long().cpu()], what="gather pairs")


def test_argmax_and_backward_vs_autograd():
    q, d, qm, dm = O.synth_colbert_inputs(3, 2, 16, 40, 64, seed=14, dtype=torch.float32, full_q=False)
    qr = q.clone().requires_grad_(True)
    dr = d.clone().requires_grad_(True)
    qe = qr.repeat_interleave(2, dim=0)
    s = torch.bmm(qe, dr.transpose(2, 1))
    s = s.masked_fill(~dm.bool().unsqueeze(1), -1000.0).max(-1).values
    s = (s * qm.repeat_interleave(2, dim=0).float()).sum(-1)
    g = torch.randn(s.shape, generator=torch.Generator().manual_seed(1))
    s.backward(g)
    from matchmaker_b200 import autograd
    cq = q.to(DEV).requires_grad_(True)
    cd = d.to(DEV).requires_grad_(True)
    out = autograd.maxsim(cq, cd, qm.to(DEV), dm.to(DEV), docs_per_query=2)
    assert_close_rel(out, s.detach(), what="fwd")
    out.backward(g.to(DEV))
    assert_close_rel(cq.grad, qr.grad, what="grad_q")
    assert_close_rel(cd.grad, dr.grad, what="grad_d")


def test_backward_is_deterministic_with_many_docs_per_query():
    """grad_q sums the contributions of a query's docs_per_query pairs: a fixed order (no atomics), so two runs agree
    bit for bit; fp16 inputs take the tensor-core forward with argmax."""
    from matchmaker_b200 import autograd
    q, d, qm, dm = O.synth_colbert_inputs(5, 300, 32, 180, 128, seed=77, full_q=False)
    g = torch.randn(5 * 300, generator=torch.Generator().manual_seed(2)).to(DEV)
    grads = []
    for _ in range(3):
        cq = q.to(DEV).requires_grad_(True)
        cd = d.to(DEV).requires_grad_(True)
        out = autograd.maxsim(cq, cd, qm.to(DEV), dm.to(DEV), docs_per_query=300)
        out.backward(g)
        grads.append((cq.grad.clone(), cd.grad.clone()))
    assert all(torch.equal(grads[0][0], x[0]) and torch.equal(grads[0][1], x[1]) for x in grads[1:])
    # against torch autograd on the upcast values
    qr = q.float().clone().requires_grad_(True)
    dr = d.float().clone().requires_grad_(True)
    s = torch.bmm(qr.repeat_interleave(300, dim=0), dr.transpose(2, 1))
    s = s.masked_fill(~dm.bool().unsqueeze(1), -1000.0).max(-1).values
    s = (s * qm.repeat_interleave(300, dim=0).float()).sum(-1)
    s.backward(g.cpu())
    assert_close_rel(grads[0][0].float(), qr.grad, rel=2e-3, what="grad_q")
    assert_close_rel(grads[0][1].float(), dr.grad, rel=2e-3, what="grad_d")


def test_baseline_size_properties():
    """BASELINE config 3 (64 queries x 1000 docs, Lq=32, Ld=180, dim=128, fp16): size-independent properties
    -- tensor cores == SIMT, permutation equivariance over documents, chunking invariance, oracle on a sample."""
    n_q, dpq = 64, 1000
    q, d, qm, dm = O.synth_colbert_inputs(n_q, dpq, 32, 180, 128, seed=1237)
    cq, cd, cqm, cdm = _cuda(q, d, qm, dm)
    s = interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=dpq, impl="tcgen05")
    assert s.shape == (n_q * dpq,) and torch.isfinite(s).all()
    s_simt = interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=dpq, impl="simt")
    assert_close_rel(s, s_simt, what="tc vs simt")
    s_docm = interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=dpq, impl="tcgen05_docm")
    assert_close_rel(s, s_docm, what="queries-on-M vs documents-on-M kernel")
    # a document's score does not depend on where it sits in the batch
    perm = torch.randperm(n_q * dpq, generator=torch.Generator().manual_seed(5)).to(DEV)
    pq = torch.div(perm, dpq, rounding_mode="floor").to(torch.int32)
    s_perm = interaction.maxsim(cq, cd, cqm, cdm, pair_q=pq, pair_d=perm.to(torch.int32), impl="tcgen05")
    assert torch.equal(s_perm, s[perm])
    # scoring a slice on its own gives the same numbers (bit-exact: same per-pair arithmetic)
    lo, hi = 17 * dpq, 19 * dpq
    s_slice = interaction.maxsim(cq[17:19], cd[lo:hi], cqm[17:19], cdm[lo:hi], docs_per_query=dpq, impl="tcgen05")
    assert torch.equal(s_slice, s[lo:hi])
    # the oracle on ALL 64 000 pairs of the config (the CPU restatement takes ~0.5 s for the whole batch)
    ref = O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, dpq)
    assert_close_rel(s, ref, what="oracle, full config 3")
    assert_close_rel(s_docm, ref, what="documents-on-M kernel vs oracle, full config 3")


def test_ragged_fetch_is_bit_identical():
    """impl="tcgen05_ragged" fetches only rows up to each document's last unmasked row; scores must not change."""
    for (n_q, dpq, Lq, Ld, dim) in [(5, 40, 32, 180, 128), (3, 7, 17, 300, 64), (2, 9, 32, 256, 128)]:
        q, d, qm, dm = O.synth_colbert_inputs(n_q, dpq, Lq, Ld, dim, seed=5 + Ld, full_q=False)
        dm[1] = 0
        dm[2, :] = 1
        dm[3, 5:] = 0
        g = torch.Generator().manual_seed(1)
        dm[4] = (torch.rand(Ld, generator=g) > 0.5).long()   # holes: last unmasked row decides
        args = _cuda(q, d, qm, dm)
        dense = interaction.maxsim(*args, docs_per_query=dpq, impl="tcgen05")
        ragged = interaction.maxsim(*args, docs_per_query=dpq, impl="tcgen05_ragged")
        assert torch.equal(dense, ragged)
        assert_close_rel(ragged, O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, dpq), what="ragged vs oracle")
        nomask = interaction.maxsim(args[0], args[1], docs_per_query=dpq, impl="tcgen05_ragged")
        assert torch.equal(nomask, interaction.maxsim(args[0], args[1], docs_per_query=dpq, impl="tcgen05"))


def test_argmax_from_the_tcgen05_epilogue_matches_the_simt_kernel():
    """Training-mode forward: the queries-on-M kernel tracks the winning document row per query token itself (autograd
    no longer drops to the SIMT kernel).  Scores bit-identical to the inference instantiation; argmax = the first maximum
    of the fp32 scores; -1 for masked query tokens, fully masked documents and maxima taken by the -1000 fill."""
    for (n_q, dpq, Lq, Ld, dim) in [(6, 50, 32, 180, 128), (3, 4, 17, 300, 64), (2, 5, 32, 77, 128)]:
        q, d, qm, dm = O.synth_colbert_inputs(n_q, dpq, Lq, Ld, dim, seed=90 + Ld, full_q=False)
        dm[1] = 0                      # fully masked document: no gradient anywhere
        dm[2, :] = 1
        # document 3: every row = -2000 x (sum of its query's tokens), so most real scores fall below the -1000 fill of its
        # masked half and the fill wins those maxima (no gradient there)
        d[3, :, :] = (-2000.0 * q[3 // dpq].float().sum(0)).to(d.dtype)
        dm[3, Ld // 2:] = 0
        args = _cuda(q, d, qm, dm)
        s_inf = interaction.maxsim(*args, docs_per_query=dpq, impl="tcgen05")
        s_trn, am = interaction.maxsim(*args, docs_per_query=dpq, impl="tcgen05", return_argmax=True)
        assert torch.equal(s_inf, s_trn)
        s_simt, am_simt = interaction.maxsim(*args, docs_per_query=dpq, impl="simt", return_argmax=True)
        # the oracle's own argmax (fp32 bmm on the upcast values), first maximum
        qe = q.float().repeat_interleave(dpq, dim=0)
        sc = torch.bmm(qe, d.float().transpose(1, 2))
        sc = sc.masked_fill(~dm.bool().unsqueeze(1), -1000.0)
        ref_max, ref_arg = sc.max(-1)
        ref_arg = ref_arg.masked_fill(~dm.bool().gather(1, ref_arg), -1)              # the fill won (or everything masked)
        ref_arg = ref_arg.masked_fill(~qm.bool().repeat_interleave(dpq, dim=0), -1)   # masked query token
        am, am_simt = am.cpu().long(), am_simt.cpu().long()
        # where the two largest scores of a row are separated beyond fp32 round-off the winner is unambiguous
        top2 = sc.topk(2, dim=-1).values
        clear = (top2[..., 0] - top2[..., 1]) > 1e-4 * top2[..., 0].abs().clamp(min=1.0)
        assert (am[clear] == ref_arg[clear]).all()
        assert (am_simt[clear] == ref_arg[clear]).all()
        assert (am[ref_arg < 0] == -1).all()
        # ragged fetch + argmax
        s_rag, am_rag = interaction.maxsim(*args, docs_per_query=dpq, impl="tcgen05_ragged", return_argmax=True)
        assert torch.equal(s_rag, s_inf) and torch.equal(am_rag.cpu().long(), am)


def test_host_buffer_pipeline_matches_device_path():
    q, d, qm, dm = O.synth_colbert_inputs(4, 250, 32, 180, 128, seed=21)
    ref = interaction.maxsim(*_cuda(q, d, qm, dm), docs_per_query=250)
    pinned = [t.pin_memory() for t in (q, d, qm, dm)]
    got = interaction.maxsim_host(*pinned, docs_per_query=250)                  # zero-copy TMA over PCIe, ragged
    assert not got.is_cuda
    assert torch.equal(got, ref.cpu())
    got_slab = interaction.maxsim_host(*pinned, docs_per_query=250, chunk_pairs=-1)  # forced staged pipeline
    assert torch.equal(got_slab, ref.cpu())
    got = interaction.maxsim_host(*pinned, docs_per_query=250, chunk_pairs=96)
    assert torch.equal(got, ref.cpu())
    got2 = interaction.maxsim_host(q, d, None, None, docs_per_query=250)  # pageable, default chunking, no masks
    assert torch.equal(got2, interaction.maxsim(*_cuda(q, d), docs_per_query=250).cpu())


def test_invalid_arguments_raise():
    q = torch.zeros(2, 32, 128, dtype=torch.float16, device=DEV)
    d = torch.zeros(5, 180, 128, dtype=torch.float16, device=DEV)
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.maxsim(q, d)  # 2 queries x 1 doc/query < 5 docs
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.maxsim(q, d.float())
    with pytest.raises(_lib.MatchmakerB200Error):
        interaction.maxsim(q.float(), d.float(), docs_per_query=3, impl="tcgen05")  # fp32 has no tcgen05 path


def test_colbert_token_index_rerank():
    """Retrieval aggregation over a resident token store (the working version of dense_retrieval.py:398-412)."""
    import numpy as np
    from matchmaker_b200.retrieval import ColBERTTokenIndex
    g = torch.Generator().manual_seed(31)
    n, dim, Lmax = 300, 128, 180
    lens = torch.randint(5, Lmax + 1, (n,), generator=g)
    mats = [torch.nn.functional.normalize(torch.randn(int(l), dim, generator=g), dim=-1).half().numpy() for l in lens]
    ext_ids = np.arange(n, dtype=np.int64) * 7 + 3
    idx = ColBERTTokenIndex(dim, Lmax)
    idx.index(ext_ids, mats)
    q = torch.nn.functional.normalize(torch.randn(4, 32, dim, generator=g), dim=-1).half()
    cand = torch.stack([torch.randperm(n, generator=g)[:50] for _ in range(4)])
    cand[2, 40:] = -1
    s, ids = idx.rerank(q, None, cand, top_n=10)
    for qi in range(4):
        ref = []
        for c in cand[qi].tolist():
            if c < 0:
                continue
            d = torch.from_numpy(mats[c]).float().unsqueeze(0)
            ref.append((O.maxsim_pairs(q[qi:qi + 1].float(), d, None, None).item(), int(ext_ids[c])))
        ref.sort(key=lambda t: (-t[0], t[1]))
        assert ids[qi].cpu().tolist() == [r[1] for r in ref[:10]]
        assert_close_rel(s[qi].cpu(), torch.tensor([r[0] for r in ref[:10]]), what="rerank scores")
