"""numpy statement of the NT GEMM descriptor (csrc/gemm_nt.cuh GemmDesc, decode_tile / epilogue in csrc/gemm_nt.cu):
which tiles a launch computes, each tile's k range, where a `sub` buffer replaces the main buffer, the diagonal mask,
the transposed copy Ct and the peer copies.  `run` applies a descriptor to named numpy buffers and returns what it read
and wrote; `decode` is a port of the kernel's rasterisation (grid index -> tile).

Coordinates follow the kernel: tile (z, bm, bn) covers C rows c_row0 + z*zstep + bm*128 + [0, 128) and columns
c_col0 + z*zstep + bn*128 + [0, 128); A rows a_row0 + z*zstep + bm*128 + i, A columns a_col0 + z*zstep + k.
"""
from dataclasses import dataclass, field

import numpy as np

BM = BN = 128
BK = 16
LOWER_ONLY, KLO_M, KHI_M, KHI_N, SKIP_FIRST, KLO_N = 1, 2, 4, 8, 16, 32
GM_TRI = 4          # gemm_nt.cu GM_TRI: group height of GEMM_KLO_M launches (16 otherwise)
BIG = 1 << 30       # gemm_desc_default(): no clipping


@dataclass
class Operand:
    buf: str
    sub: str = None          # compact [Npad x 128] buffer of clean diagonal tiles
    row0: int = 0
    col0: int = 0


@dataclass
class Desc:
    A: Operand
    B: Operand
    C: str
    M: int
    N: int
    K: int
    c_row0: int = 0
    c_col0: int = 0
    Ct: str = None
    ct_row0: int = 0
    ct_col0: int = 0
    alpha: float = 1.0
    beta: float = 0.0
    flags: int = 0
    batch: int = 1
    zstep: int = 0
    m_lim: int = BIG
    n_lim: int = BIG
    k_lim: int = BIG
    klo_off: int = 0
    bm_mod: int = 0
    bm_rem: int = 0
    bn_mod: int = 0
    bn_rem: int = 0
    bm_div: int = 0
    bm_off: int = 0
    bn_div: int = 0
    bn_off: int = 0
    peers: tuple = field(default_factory=tuple)


@dataclass
class Tile:
    z: int
    bm: int
    bn: int
    klo: int      # k range [klo, khi) in elements (empty when khi <= klo: the tile still writes beta * C)
    khi: int


def _div(v):
    return v if v > 0 else 1


def owned(d, bm, bn):
    ok_m = d.bm_mod <= 1 or ((bm + d.bm_off) // _div(d.bm_div)) % d.bm_mod == d.bm_rem
    ok_n = d.bn_mod <= 1 or ((bn + d.bn_off) // _div(d.bn_div)) % d.bn_mod == d.bn_rem
    return ok_m and ok_n


def k_range(d, z, bm, bn):
    Kz = min(d.K, d.k_lim - z * d.zstep)
    lo = (d.klo_off + bm * BM) // BK if d.flags & KLO_M else 0
    if d.flags & KLO_N:
        lo = max(lo, bn * (BN // BK))
    hi = Kz // BK if Kz > 0 else 0
    if d.flags & KHI_M:
        hi = min(hi, (bm + 1) * (BM // BK))
    if d.flags & KHI_N:
        hi = min(hi, (bn + 1) * (BN // BK))
    return lo * BK, hi * BK


def tiles(d):
    """Every tile the launch computes, in (z, bm, bn) order."""
    out = []
    tm, tn = d.M // BM, d.N // BN
    for z in range(d.batch):
        Mz = min(d.M, d.m_lim - z * d.zstep)
        Nz = min(d.N, d.n_lim - z * d.zstep)
        for bm in range(tm):
            for bn in range(tn):
                if bm * BM >= Mz or bn * BN >= Nz:
                    continue
                if d.flags & LOWER_ONLY and bn > bm:
                    continue
                if d.flags & SKIP_FIRST and bm == 0 and bn == 0:
                    continue
                if not owned(d, bm, bn):
                    continue
                out.append(Tile(z, bm, bn, *k_range(d, z, bm, bn)))
    return out


# ---- rasterisation (decode_tile) ---------------------------------------------------------------------------------

def _own_before(d, t):
    div = _div(d.bm_div)
    cyc = div * d.bm_mod
    c, r = divmod(t, cyc)
    return c * div + min(max(r - d.bm_rem * div, 0), div)


def grid_size(d):
    """gridDim.x of gemm_nt_launch (0: nothing launched)."""
    tm, tn = d.M // BM, d.N // BN
    n = tm * tn
    if d.flags & LOWER_ONLY:
        n = sum(min(r, tn - 1) + 1 for r in range(tm))
    if d.bm_mod > 1 and d.batch == 1:
        first = _own_before(d, d.bm_off)
        n_own = _own_before(d, d.bm_off + tm) - first
        n = 0 if n_own <= 0 else (n_own + 7) // 8 * 8 * tn
    return n


def decode(d, lin):
    """(bm, bn) the CTA with blockIdx.x = lin works on, before the validity test (port of decode_tile)."""
    tm, tn = d.M // BM, d.N // BN
    GM = GM_TRI if d.flags & KLO_M else 16
    rem = lin
    if d.bm_mod > 1 and d.batch == 1:
        div = _div(d.bm_div)
        first = _own_before(d, d.bm_off)
        n_own = _own_before(d, d.bm_off + tm) - first
        group, in_group = divmod(rem, 8 * tn)
        o = group * 8 + in_group % 8
        bn = in_group // 8
        if o >= n_own:
            return tm, bn
        og = o + first
        return ((og // div) * d.bm_mod + d.bm_rem) * div + og % div - d.bm_off, bn
    if not d.flags & LOWER_ONLY:
        per = GM * tn
        group = rem // per
        first = group * GM
        gs = min(GM, tm - first)
        ing = rem - group * per
        return first + ing % gs, ing // gs
    first = 0
    while True:
        gs = min(GM, tm - first)
        cnt = sum(min(r, tn - 1) + 1 for r in range(first, first + gs))
        if rem < cnt or first + gs >= tm:
            break
        rem -= cnt
        first += gs
    full = min(first, tn)
    if rem < full * gs:
        return first + rem % gs, rem // gs
    rem -= full * gs
    bn = full
    while True:
        nrows = first + gs - max(bn, first)
        if rem < nrows or bn + 1 >= tn:
            break
        rem -= nrows
        bn += 1
    return max(bn, first) + rem, bn


def rasterised_tiles(d):
    """The (z, bm, bn) set the launched grid computes: decode every CTA and apply decode_tile's validity test."""
    have = {(t.z, t.bm, t.bn) for t in tiles(d)}
    out = []
    tm, tn = d.M // BM, d.N // BN
    for z in range(d.batch):
        Mz = min(d.M, d.m_lim - z * d.zstep)
        Nz = min(d.N, d.n_lim - z * d.zstep)
        for lin in range(grid_size(d)):
            bm, bn = decode(d, lin)
            valid = (bm * BM < Mz and bn * BN < Nz and (not d.flags & LOWER_ONLY or bn <= bm)
                     and (not d.flags & SKIP_FIRST or bm or bn) and owned(d, bm, bn))
            if valid:
                assert 0 <= bm < tm and 0 <= bn < tn, (lin, bm, bn)
                out.append((z, bm, bn))
    return out, have


# ---- semantics ---------------------------------------------------------------------------------------------------

def _operand_rows(d, op, z, b, k0, k1):
    """Per k-step [ks, ks+16) of [k0, k1): (buffer name, row slice, column slice) the tile reads for operand rows b*128.."""
    zo = z * d.zstep
    r = op.row0 + zo + b * BM
    out = []
    for ks in range(k0, k1, BK):
        c = op.col0 + zo + ks
        if op.sub is not None and (c >> 7) == (r >> 7):
            out.append((op.sub, slice(r, r + BM), slice(c & 127, (c & 127) + BK)))
        else:
            out.append((op.buf, slice(r, r + BM), slice(c, c + BK)))
    return out


def run(d, bufs, acc_dtype=np.float64):
    """Apply launch `d` to the dict of 2-D arrays `bufs` (in place).  Returns (read, written): dicts name -> bool mask.
    Every tile reads the launch's inputs as they were before the launch; a descriptor where one tile stores an element
    another tile reads as A / B (a race on the device) raises.  A tile may overwrite its own operand (in-place TRSM)."""
    snap = {k: v.copy() for k, v in bufs.items()}
    read_by = {k: np.full(v.shape, -1) for k, v in bufs.items()}       # tile index reading it as A / B, -2: several
    written = {k: np.zeros(v.shape, bool) for k, v in bufs.items()}
    c_read = {k: np.zeros(v.shape, bool) for k, v in bufs.items()}
    results = []
    for i, t in enumerate(tiles(d)):
        acc = np.zeros((BM, BN), acc_dtype)
        for (na, ra, ca), (nb, rb, cb) in zip(_operand_rows(d, d.A, t.z, t.bm, t.klo, t.khi),
                                              _operand_rows(d, d.B, t.z, t.bn, t.klo, t.khi)):
            a = snap[na][ra, ca]
            b = snap[nb][rb, cb]
            assert a.shape == (BM, BK) and b.shape == (BN, BK), "operand outside its buffer"
            for n, r, c in ((na, ra, ca), (nb, rb, cb)):
                v = read_by[n][r, c]
                v[(v != -1) & (v != i)] = -2
                v[v == -1] = i
            acc += a.astype(acc_dtype) @ b.astype(acc_dtype).T
        zo = t.z * d.zstep
        rc = slice(d.c_row0 + zo + t.bm * BM, d.c_row0 + zo + (t.bm + 1) * BM)
        cc = slice(d.c_col0 + zo + t.bn * BN, d.c_col0 + zo + (t.bn + 1) * BN)
        v = acc_dtype(d.alpha) * acc
        if d.beta != 0.0:
            v = v + acc_dtype(d.beta) * snap[d.C][rc, cc].astype(acc_dtype)
            c_read[d.C][rc, cc] = True
        mask = np.ones((BM, BN), bool)
        if d.flags & LOWER_ONLY and t.bm == t.bn:
            mask = np.tril(mask)
        results.append((i, d.C, rc, cc, v, mask))
        for p in d.peers:
            results.append((i, p, rc, cc, v, mask))
        if d.Ct is not None:
            rt = slice(d.ct_row0 + zo + t.bn * BN, d.ct_row0 + zo + (t.bn + 1) * BN)
            ct = slice(d.ct_col0 + zo + t.bm * BM, d.ct_col0 + zo + (t.bm + 1) * BM)
            results.append((i, d.Ct, rt, ct, v.T, mask.T))
    for i, name, r, c, v, mask in results:
        tgt = bufs[name][r, c]
        assert tgt.shape == v.shape, "store outside its buffer"
        assert not (written[name][r, c] & mask).any(), "two tiles store the same element"
        rb = read_by[name][r, c][mask]
        assert ((rb == -1) | (rb == i)).all(), "a tile stores an element another tile reads (%s)" % name
        tgt[mask] = v[mask]
        written[name][r, c] |= mask
    read = {k: (read_by[k] != -1) | c_read[k] for k in bufs}
    return read, written
