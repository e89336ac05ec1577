"""Index model of the data-movement kernels of the multi-rank schedules (csrc/shard_kernels.cuh), in plain Python / numpy.

Row-sharded storage deals 128-row tiles block-cyclically: tile t belongs to rank (t // rb) % R.  A rank's "compact"
vectors hold one entry per own row, own tiles in ascending order.  Replicated storage (inverse_dist) splits a level s
of the triangular inverse by 128-wide tile columns of every W21 block: rank q computes the tile columns t % R == q."""
import numpy as np

T = 128

# the ownership layouts (R, rb) the tests sweep, and the tile counts per layout
LAYOUTS = [(1, 1), (2, 1), (3, 2), (4, 1), (5, 3), (8, 1), (2, 8), (8, 2)]


def tile_counts(R, rb):
    """1, a cycle short by one, a full cycle, one tile into the next, three cycles and a partial fourth"""
    c = R * rb
    return sorted({n for n in (1, c - 1, c, c + 1, 3 * c + 2) if n >= 1})


def owner(t, R, rb):
    return (t // rb) % R


def own_before(t, q, R, rb):
    """number of tiles t' < t owned by rank q (shard_own_before)"""
    cyc = rb * R
    c, rem = divmod(t, cyc)
    return c * rb + min(max(rem - q * rb, 0), rb)


def own_tiles(n_tiles, me, R, rb, t1=0):
    return [t for t in range(t1, n_tiles) if owner(t, R, rb) == me]


def compact_rows(n_tiles, me, R, rb, t1=0):
    """global row of every compact index li among the own rows of tiles t1 .. n_tiles (ascending)"""
    ts = own_tiles(n_tiles, me, R, rb, t1)
    if not ts:
        return np.zeros(0, np.int64)
    return (np.asarray(ts, np.int64)[:, None] * T + np.arange(T)[None, :]).ravel()


def own_row_mask(nrows, me, R, rb):
    return owner(np.arange(nrows) // T, R, rb) == me


def own_rows(n, me, R, rb):
    """length of the compact vectors of the rows 0 .. n (shard_own_rows)"""
    return own_before(-(-n // T), me, R, rb) * T


# ---- replicated storage: inverse_dist's column slices ----------------------------------------------------------------

def split_levels(Np, R):
    """the levels s of the triangular inverse that inverse_dist splits over R ranks"""
    out, s = [], T
    while s < Np:
        tiles = s // T
        if tiles >= R and tiles % R == 0:
            out.append(s)
        s *= 2
    return out


def problems(s, Np):
    """(z, p, n2) of every problem of level s that has a W21 block (n2 > 0)"""
    batch = -(-Np // (2 * s))
    out = []
    for z in range(batch):
        p = 2 * s * z
        n2 = min(s, Np - p - s)
        if n2 > 0:
            out.append((z, p, n2))
    return out


def slice_cols(s, R, q):
    """block column gj of every local column jl of rank q's slice (wr = s / R columns)"""
    jl = np.arange(s // R)
    return ((jl // T) * R + q) * T + jl % T


def per_rank(s, Np, R):
    """doubles per rank of the all-gather, sum_z n2_z * wr, as inverse_dist computes it"""
    return sum(n2 for _, _, n2 in problems(s, Np)) * (s // R)
