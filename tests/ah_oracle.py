"""CPU fp64 restatement of the AH (ScaNN-style) index: nibble packing, the anisotropic loss and its weight, the lookup
tables, the approximate scan over the probed leaves and the exact reorder of the shortlist."""
import torch

NO_RESULT = -3.4028234663852886e38


def eta(dim, threshold=0.2):
    return (dim - 1) * threshold ** 2 / (1 - threshold ** 2)


def pack(codes):
    """[n, M] in 0..15 -> [n, M/2] uint8, block 2j low nibble, 2j + 1 high nibble, by a loop over bytes."""
    n, M = codes.shape
    out = torch.zeros((n, M // 2), dtype=torch.uint8)
    for j in range(M // 2):
        out[:, j] = (codes[:, 2 * j] + 16 * codes[:, 2 * j + 1]).to(torch.uint8)
    return out


def unpack(packed):
    p = packed.to(torch.int64)
    n, B = p.shape
    out = torch.zeros((n, 2 * B), dtype=torch.int64)
    for j in range(B):
        out[:, 2 * j], out[:, 2 * j + 1] = p[:, j] % 16, p[:, j] // 16
    return out


def loss(r, x, codebook, codes, eta_):
    """Per-row |e|^2 + (eta - 1) (e . x/|x|)^2 with e = r - r~ (x = 0: the plain loss), fp64."""
    M = codebook.shape[0]
    rt = torch.stack([codebook[m, codes[:, m]] for m in range(M)], dim=1).reshape(r.shape[0], -1).double()
    e = r.double() - rt
    nrm = x.double().norm(dim=1, keepdim=True)
    xh = torch.where(nrm > 0, x.double() / nrm.clamp_min(1e-300), torch.zeros_like(nrm))
    return (e * e).sum(1) + (eta_ - 1) * (e * xh).sum(1) ** 2


def luts(q, codebook):
    """[nq, M, 16] fp64: T[m][j] = q[2m] C[m][j][0] + q[2m+1] C[m][j][1]."""
    qd, c = q.double(), codebook.double()
    return qd[:, 0::2].unsqueeze(2) * c[:, :, 0].unsqueeze(0) + qd[:, 1::2].unsqueeze(2) * c[:, :, 1].unsqueeze(0)


def _order(score, key):
    """Indices sorting by (score desc, key asc): two stable sorts."""
    o = torch.sort(key, stable=True).indices
    return o[torch.sort(-score[o], stable=True).indices]


def scan(tables, packed, offsets, probes, bias, kr):
    """(scores [nq, kr], row positions [nq, kr]): the kr best rows of the probed leaves by bias + sum_m T[m][code_m]
    (fp64) under (score desc, position asc), (-FLT_MAX, -1) tail.  Leaf ids outside [0, nlist) probe nothing."""
    codes = unpack(packed)
    nq = probes.shape[0]
    nlist = offsets.numel() - 1
    M = codes.shape[1]
    out_s = torch.full((nq, kr), NO_RESULT, dtype=torch.float64)
    out_p = torch.full((nq, kr), -1, dtype=torch.int64)
    for q in range(nq):
        t = tables[q].double()
        s_parts, p_parts = [], []
        for j, l in enumerate(probes[q].tolist()):
            if not 0 <= l < nlist:
                continue
            pos = torch.arange(int(offsets[l]), int(offsets[l + 1]))
            if pos.numel() == 0:
                continue
            sc = t[torch.arange(M).unsqueeze(0), codes[pos]].sum(1) + float(bias[q, j])
            s_parts.append(sc)
            p_parts.append(pos)
        if not s_parts:
            continue
        s, p = torch.cat(s_parts), torch.cat(p_parts)
        order = _order(s, p)[:kr]
        out_s[q, :len(order)] = s[order]
        out_p[q, :len(order)] = p[order]
    return out_s, out_p


def reorder(q, rows, ids, shortlist, top_n):
    """Exact fp64 inner products of each query with its shortlisted rows (positions < 0 are void), the top_n under
    (score desc, id asc), (-FLT_MAX, -1) tail."""
    nq = q.shape[0]
    out_s = torch.full((nq, top_n), NO_RESULT, dtype=torch.float64)
    out_i = torch.full((nq, top_n), -1, dtype=torch.int64)
    for a in range(nq):
        pos = shortlist[a][shortlist[a] >= 0]
        if pos.numel() == 0:
            continue
        s = rows[pos].double() @ q[a].double()
        uid = ids[pos]
        order = _order(s, uid)[:top_n]
        out_s[a, :len(order)] = s[order]
        out_i[a, :len(order)] = uid[order]
    return out_s, out_i


def scan_slots(tables, packed, offsets, probes, bias, kr, kslot):
    """scan() when each (query, probe) keeps only its kslot best rows before the merge: what the kernel returns for a
    leaf longer than the max_list_len it was given."""
    nq = probes.shape[0]
    out_s = torch.full((nq, kr), NO_RESULT, dtype=torch.float64)
    out_p = torch.full((nq, kr), -1, dtype=torch.int64)
    for q in range(nq):
        s_parts, p_parts = [], []
        for j in range(probes.shape[1]):
            s, p = scan(tables[q:q + 1], packed, offsets, probes[q:q + 1, j:j + 1], bias[q:q + 1, j:j + 1], kslot)
            s_parts.append(s[0][p[0] >= 0])
            p_parts.append(p[0][p[0] >= 0])
        s, p = torch.cat(s_parts), torch.cat(p_parts)
        order = _order(s, p)[:kr]
        out_s[q, :len(order)] = s[order]
        out_p[q, :len(order)] = p[order]
    return out_s, out_p
