"""numpy restatement of the residual token code format (matchmaker_b200/csrc/residual.cuh, DESIGN 3.4g).

Row x of list l: code[d] = #{i : cutoff[d][i] <= float32(x[d]) - float32(base[l][d])}, decoded value
fp16_rn(float32(base[l][d]) + float32(weight[d][code[d]])); dimension d in bits [b * (d % (8 / b)), +b) of byte
d * b / 8."""
import numpy as np


def pack(codes, bits):
    """[n, dim] codes in [0, 2^bits) -> [n, dim * bits / 8] uint8."""
    n, dim = codes.shape
    per = 8 // bits
    c = codes.reshape(n, dim // per, per).astype(np.uint32)
    return (c << (bits * np.arange(per, dtype=np.uint32))).sum(-1).astype(np.uint8)


def unpack(packed, bits, dim):
    per = 8 // bits
    p = packed.astype(np.uint32)[:, :, None] >> (bits * np.arange(per, dtype=np.uint32))
    return (p & ((1 << bits) - 1)).reshape(packed.shape[0], dim).astype(np.uint8)


def residuals(rows, list_ids, base):
    return rows.astype(np.float32) - base[list_ids].astype(np.float32)


def codes(rows, list_ids, base, cutoff):
    """Unpacked codes [n, dim] (cutoff [dim, 2^b - 1] fp32)."""
    r = residuals(rows, list_ids, base)
    return (cutoff[None, :, :] <= r[:, :, None]).sum(-1).astype(np.uint8)


def encode(rows, list_ids, base, cutoff, bits):
    return pack(codes(rows, list_ids, base, cutoff), bits)


def decode(packed, list_ids, base, weight, bits):
    dim = base.shape[1]
    c = unpack(packed, bits, dim)
    w = weight[np.arange(dim)[None, :], c]
    return (base[list_ids].astype(np.float32) + w.astype(np.float32)).astype(np.float16)


def quantile_tables(r, bits):
    """(cutoff [dim, 2^b - 1] fp32, weight [dim, 2^b] fp16): nearest-rank i / 2^b and (i + 0.5) / 2^b quantiles of the
    residuals r [n, dim] (ColBERTResidualIndexer.train_tables)."""
    rs = np.sort(r.astype(np.float32), axis=0)
    n, nlev = r.shape[0], 1 << bits

    def pick(fr):
        return rs[min(n - 1, int(fr * n))]
    cutoff = np.stack([pick(i / nlev) for i in range(1, nlev)], axis=1).astype(np.float32)
    weight = np.stack([pick((i + 0.5) / nlev) for i in range(nlev)], axis=1).astype(np.float16)
    return cutoff, weight


def synth(n, dim, nlist, bits, seed):
    """Rows, list ids, fp16 bases (list 0 zero, the last list with large-norm rows), tables from the residuals, and
    some residuals placed exactly on a cutoff."""
    rng = np.random.default_rng(seed)
    base = (rng.standard_normal((nlist, dim)) * 0.3).astype(np.float16)
    base[0] = 0
    lids = rng.integers(0, nlist, n).astype(np.int32)
    rows = (base[lids].astype(np.float32) + rng.standard_normal((n, dim)) * 0.1).astype(np.float16)
    big = lids == nlist - 1
    rows[big] = (rows[big].astype(np.float32) * 200.0).astype(np.float16)
    cutoff, weight = quantile_tables(residuals(rows, lids, base), bits)
    # rows of list 0 (zero base) hit the cutoffs exactly: the residual is the fp16 row itself
    z = np.nonzero(lids == 0)[0][:8]
    for j, r in enumerate(z):
        d = np.arange(dim)
        cut = cutoff[d, j % cutoff.shape[1]].astype(np.float16)
        rows[r] = cut
        cutoff[d, j % cutoff.shape[1]] = cut.astype(np.float32)
    cutoff = np.sort(cutoff, axis=1)
    return rows, lids, base, cutoff, weight
