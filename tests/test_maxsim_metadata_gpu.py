"""The per-pair metadata pipeline of the queries-on-M max-sim kernel: indices, lengths and mask words are fetched
ahead of use (32 pairs per batch, the mask words of a writer's next tiles in flight), so the places where a look-ahead
can go wrong are tested here: per-CTA pair ranges that are not multiples of the batch, fewer pairs than SMs, one pair
per CTA, the query changing inside a batch, every mask element type, mask views at an unaligned storage offset, Ld that
is not 16-byte aligned and Ld > 255 (two tiles), dim 64, bf16, the pair_d / pair_dmask indirection, the argmax
instantiation and store mode with empty passages and skipped pairs.

Dense fetch, ragged fetch and store mode must agree bit for bit on the same data; the oracle within the parity bar."""
import pytest
import torch

from conftest import assert_close_rel
from matchmaker_b200 import interaction
from oracle import interaction_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"

SHAPES = [  # n_q, docs_per_query, Lq, Ld, dim, dtype
    (1, 100, 32, 180, 128, torch.float16),     # fewer pairs than SMs
    (1, 132, 32, 180, 128, torch.float16),     # one pair per CTA
    (400, 1, 32, 181, 128, torch.float16),     # a new query every pair; 3-4 pairs per CTA; Ld not 16-B aligned
    (3, 1000, 17, 7, 64, torch.bfloat16),      # dim 64, bf16, tiny documents, query changes inside a batch
    (47, 3, 32, 300, 128, torch.float16),      # two tiles per document
    (20, 1000, 32, 180, 128, torch.float16),   # 151-152 pairs per CTA
    (2, 150, 32, 220, 128, torch.float16),     # 256-row tile (NCH = 4): the widest writer register sets
    (3, 60, 32, 100, 64, torch.bfloat16),      # 128-row tile (NCH = 2)
]


def _masks_with_edge_documents(dm, Ld):
    dm[0] = 0                       # fully masked
    dm[min(1, dm.shape[0] - 1), :] = 1
    g = torch.Generator().manual_seed(3)
    dm[dm.shape[0] // 2] = (torch.rand(Ld, generator=g) > 0.5).long()   # holes
    return dm


@pytest.mark.parametrize("shape", SHAPES)
def test_dense_ragged_and_oracle_agree(shape):
    n_q, dpq, Lq, Ld, dim, dt = shape
    q, d, qm, dm = O.synth_colbert_inputs(n_q, dpq, Lq, Ld, dim, seed=300 + Ld + dpq, dtype=dt, full_q=False)
    dm = _masks_with_edge_documents(dm, Ld)
    cq, cd, cqm, cdm = (t.to(DEV) for t in (q, d, qm, dm))
    dense = interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=dpq, impl="tcgen05")
    ragged = interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=dpq, impl="tcgen05_ragged")
    assert torch.equal(dense, ragged)
    assert_close_rel(dense, O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, dpq), what=str(shape))
    s_trn, am = interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=dpq, impl="tcgen05", return_argmax=True)
    s_rag, am_rag = interaction.maxsim(cq, cd, cqm, cdm, docs_per_query=dpq, impl="tcgen05_ragged", return_argmax=True)
    assert torch.equal(s_trn, dense) and torch.equal(s_rag, dense) and torch.equal(am, am_rag)


@pytest.mark.parametrize("mdt", [torch.bool, torch.uint8, torch.int32, torch.int64, torch.float32])
def test_mask_dtypes_as_offset_views(mdt):
    n_q, dpq, Lq, Ld, dim = 5, 61, 32, 181, 128
    q, d, qm, dm = O.synth_colbert_inputs(n_q, dpq, Lq, Ld, dim, seed=11, full_q=False)
    dm = _masks_with_edge_documents(dm, Ld)
    # views into larger tensors: the mask rows start at a non-zero storage offset, not 16-byte aligned
    big_dm = torch.zeros(dm.shape[0] + 3, Ld, dtype=mdt, device=DEV)
    big_dm[3:] = dm.to(DEV).to(mdt)
    big_qm = torch.zeros(n_q + 1, Lq, dtype=mdt, device=DEV)
    big_qm[1:] = qm.to(DEV).to(mdt)
    vqm, vdm = big_qm[1:], big_dm[3:]
    assert vdm.storage_offset() > 0 and vdm.is_contiguous()
    cq, cd = q.to(DEV), d.to(DEV)
    dense = interaction.maxsim(cq, cd, vqm, vdm, docs_per_query=dpq, impl="tcgen05")
    ragged = interaction.maxsim(cq, cd, vqm, vdm, docs_per_query=dpq, impl="tcgen05_ragged")
    ref_masks = interaction.maxsim(cq, cd, qm.to(DEV).bool(), dm.to(DEV).bool(), docs_per_query=dpq, impl="tcgen05")
    assert torch.equal(dense, ragged) and torch.equal(dense, ref_masks)
    assert_close_rel(dense, O.maxsim_one_query_many_docs(q.float(), d.float(), qm, dm, dpq), what=str(mdt))


@pytest.mark.parametrize("n", [7, 40])
def test_pair_indirection_allpairs(n):
    """pair_q / pair_d / pair_dmask: the index arrays are batch-loaded and the mask row is a second-level load."""
    Lq, Ld, dim = 32, 181, 128
    q, _, qm, _ = O.synth_colbert_inputs(n, 1, Lq, Ld, dim, seed=21 + n, full_q=False)
    _, d, _, dm = O.synth_colbert_inputs(n, 1, Lq, Ld, dim, seed=22 + n, full_q=False)
    dm = _masks_with_edge_documents(dm, Ld)
    cq, cd, cqm, cdm = (t.to(DEV) for t in (q, d, qm, dm))
    own = interaction.maxsim_allpairs(cq, cqm, cd, cdm, impl="tcgen05")
    assert_close_rel(own, O.maxsim_allpairs_own_masks(q.float(), qm, d.float(), dm), what="allpairs own masks")
    refi = interaction.maxsim_allpairs(cq, cqm, cd, cdm, impl="tcgen05", reference_mask_indexing=True)
    assert_close_rel(refi, O.maxsim_allpairs(q.float(), qm, d.float(), dm), what="allpairs reference mask indexing")
    # a shuffled pair list scores each pair as the dense layout does
    g = torch.Generator().manual_seed(n)
    perm = torch.randperm(n * n, generator=g)
    pq = (perm // n).to(torch.int32).to(DEV)
    pd = (perm % n).to(torch.int32).to(DEV)
    got = interaction.maxsim(cq, cd, cqm, cdm, pair_q=pq, pair_d=pd, impl="tcgen05")
    assert torch.equal(got, own.view(-1)[perm.to(DEV)])


def test_store_mode_matches_padded_layout():
    """Store mode with empty passages and pair_d < 0: the passage lengths come from doc_offsets (second-level loads)."""
    Lq, Ld, dim, n_docs, n_q = 32, 180, 128, 500, 9
    g = torch.Generator().manual_seed(77)
    lens = torch.randint(0, Ld + 1, (n_docs,), generator=g)
    lens[::37] = 0                                  # empty passages
    off = torch.zeros(n_docs + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(lens, 0)
    store = torch.nn.functional.normalize(torch.randn(int(off[-1]), dim, generator=g), dim=-1).half()
    q = torch.nn.functional.normalize(torch.randn(n_q, Lq, dim, generator=g), dim=-1).half()
    n_pairs = 1001
    pair_q = torch.randint(0, n_q, (n_pairs,), generator=g).sort().values.to(torch.int32)
    pair_d = torch.randint(0, n_docs, (n_pairs,), generator=g).to(torch.int32)
    pair_d[::13] = -1                               # skipped pairs
    # the same pairs in the padded layout: document p of the padded tensor is pair p's passage
    pos = torch.arange(Ld)
    dd = pair_d.clamp(min=0).long()
    plen = torch.where(pair_d >= 0, lens[dd], torch.zeros_like(lens[dd]))
    mask = pos.unsqueeze(0) < plen.unsqueeze(1)
    rows = (off[dd].unsqueeze(1) + pos.unsqueeze(0)).clamp(max=store.shape[0] - 1)
    padded = store[rows] * mask.unsqueeze(-1).half()
    dev = [t.to(DEV) for t in (q, store, off, pair_q, pair_d, padded, mask)]
    cq, cstore, coff, cpq, cpd, cpad, cmask = dev
    s_store = interaction.maxsim_store(cq, cstore, coff, cpq, cpd, Ld)
    s_pad = interaction.maxsim(cq, cpad, None, cmask, pair_q=cpq, pair_d=torch.arange(n_pairs, dtype=torch.int32,
                                                                                          device=DEV), impl="tcgen05")
    real = (plen > 0).to(DEV)
    assert torch.isinf(s_store[~real]).all() and (s_store[~real] < 0).all()
    assert torch.equal(s_store[real], s_pad[real])
    ref = O.maxsim_pairs(q.float()[pair_q.long()], padded.float(), None, mask)
    assert_close_rel(s_store[real], ref[real.cpu()], what="store mode vs oracle")
