"""Numpy restatements of csrc/pairgen.cu's random streams and of usip_cloud_subsample's selection rule, for exact
comparison with both subset kernels.

philox4x32_10 is common.cuh's Philox4x32-10 (Salmon et al., SC'11) on uint32 arrays; pg_random builds pairgen.cu's
counter (item, cloud, step, purpose | sub << 8 | step_hi << 16) and key (seed_lo, seed_hi).  subset_rows states the
header's contract for level 0: the N smallest (31-bit key, row) pairs among the rows inside the radius, ascending, or
every valid row t times then the remainder, or rows 0 without a valid row."""
import numpy as np

PURPOSE_ROWS, PURPOSE_CAND, PURPOSE_START = 0, 1, 2
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Ten rounds on uint32 counter words (broadcast arrays) and a scalar key -> four uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & _LO for x in np.broadcast_arrays(c0, c1, c2, c3)]
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & _LO
        hi1, lo1 = p1 >> np.uint64(32), p1 & _LO
        c = [hi1 ^ c[1] ^ np.uint64(k0), lo1, hi0 ^ c[3] ^ np.uint64(k1), lo0]
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return [x.astype(np.uint32) for x in c]


def pg_random(seed, step, cloud, item, purpose, sub=0):
    """pairgen.cu pg_random for an array of items -> four uint32 arrays."""
    seed, step = int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1)
    item = np.asarray(item, dtype=np.uint64)
    c3 = (purpose | (sub << 8) | ((step >> 32) << 16)) & 0xFFFFFFFF
    return philox4x32_10(item, cloud, step & 0xFFFFFFFF, c3, seed, seed >> 32)


def subset_keys(seed, step, cloud, n, purpose, ok=None):
    """pg_subset_key for items 0..n-1: the 31-bit keys, 0xffffffff where ok is False."""
    k = np.empty(n, np.uint32)
    for i in range(0, n, 1 << 22):                # bounded temporaries at 2^24 rows
        k[i:i + (1 << 22)] = pg_random(seed, step, cloud, np.arange(i, min(n, i + (1 << 22))), purpose)[0] >> 1
    if ok is not None:
        k = np.where(ok, k, np.uint32(0xFFFFFFFF))
    return k


def inside(xyz, radius):
    """pg_inside: sqrt(fl32(fl32(x*x) + fl32(z*z))) in fp32, compared in double."""
    x, z = xyz[:, 0].astype(np.float32), xyz[:, 2].astype(np.float32)
    return np.sqrt(x * x + z * z).astype(np.float64) <= radius


def _smallest(keys, idx, need):
    """The need smallest (key, index) pairs of keys[idx], as ascending indices."""
    order = np.lexsort((idx, keys[idx]))
    return np.sort(idx[order[:need]])


def subset_rows(scan, N, seed, step, cloud, radius=None):
    """Level 0 of usip_cloud_subsample for one cloud -> (rows (N,) int32, valid)."""
    n = len(scan)
    ok = np.ones(n, bool) if radius is None else inside(scan, radius)
    valid = np.flatnonzero(ok)
    nv = len(valid)
    if nv == 0:
        return np.zeros(N, np.int32), 0
    keys = subset_keys(seed, step, cloud, n, PURPOSE_ROWS, ok)
    if nv >= N:
        return _smallest(keys, valid, N).astype(np.int32), nv
    tiles = max(1, -(-N // nv) - 1)
    rest = _smallest(keys, valid, N - tiles * nv)
    return np.concatenate([np.tile(valid, tiles), rest]).astype(np.int32), nv


def subset_candidates(N, n_cand, seed, step, cloud):
    """Level 1 for one cloud -> (cand (n_cand,) int32 ascending positions into the rows, FPS start)."""
    keys = subset_keys(seed, step, cloud, N, PURPOSE_CAND)
    cand = _smallest(keys, np.arange(N), n_cand).astype(np.int32)
    r = int(pg_random(seed, step, cloud, [0], PURPOSE_START)[0][0])
    return cand, (r * n_cand) >> 32
