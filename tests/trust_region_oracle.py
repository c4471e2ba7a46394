"""numpy restatement of the device trust-region candidate source (DESIGN.md 4.18, csrc/select.cuh philox_tr_coord).

Per (seed, global row r, column j):
    u_j  = oracle.gp_oracle.philox_uniform over [lo, hi]      (counter (r_lo, r_hi, j/2, 0))
    v_j  = the same 53-bit uniform from counter (r_lo, r_hi, j/2, 1)
    f(r) = (o0 * d) >> 32, o0 the first word of counter (r_lo, r_hi, 0, 2)
    x_j  = (j == f(r) || v_j < p) ? u_j : center_j
It sits next to the other test oracles and builds on oracle.gp_oracle's Philox4x32-10, which it does not change.
"""
import numpy as np

from oracle.gp_oracle import philox4x32_10, philox_uniform

_M32 = np.uint64(0xFFFFFFFF)


def _lane_uniform(seed, rows, d, lane):
    """(len(rows), d) 53-bit uniforms of counter lane 3 = lane, with philox_uniform's word layout."""
    rows = np.asarray(rows, dtype=np.int64).astype(np.uint64)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    out = np.empty((len(rows), d))
    with np.errstate(over="ignore"):
        for b in range((d + 1) // 2):
            o = philox4x32_10(rows & _M32, rows >> np.uint64(32), np.full(len(rows), b, dtype=np.uint64),
                              np.full(len(rows), lane, dtype=np.uint64), seed & 0xFFFFFFFF, seed >> 32)
            for half in range(2):
                j = 2 * b + half
                if j >= d:
                    break
                w = o[2 * half] | (o[2 * half + 1] << np.uint64(32))
                out[:, j] = (w >> np.uint64(11)).astype(np.float64) * 2.0**-53
    return out


def forced_column(seed, rows, d):
    """(len(rows),) f(r) = (o0 * d) >> 32 of counter (r_lo, r_hi, 0, 2)."""
    rows = np.asarray(rows, dtype=np.int64).astype(np.uint64)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    with np.errstate(over="ignore"):
        o0 = philox4x32_10(rows & _M32, rows >> np.uint64(32), np.zeros(len(rows), dtype=np.uint64),
                           np.full(len(rows), 2, dtype=np.uint64), seed & 0xFFFFFFFF, seed >> 32)[0]
    return ((o0 * np.uint64(d)) >> np.uint64(32)).astype(np.int64)


def philox_tr(seed, rows, d, lo, hi, center, p):
    """Rows `rows` (global indices) of the trust-region source: (len(rows), d)."""
    u = philox_uniform(seed, rows, d, lo, hi)
    if p >= 1.0:
        return u
    v = _lane_uniform(seed, rows, d, 1)
    f = forced_column(seed, rows, d)
    mask = (v < p) | (np.arange(d)[None, :] == f[:, None])
    return np.where(mask, u, np.asarray(center, dtype=np.float64)[None, :])
