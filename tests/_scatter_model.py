"""Model of the discrete steps of reassignment and synchrosqueezing (kernels/reassign.cu, kernels/squeeze.cu), run on
GIVEN float32 planes.

The float64 oracle computes a cell's destination from float64 spectra, so near a rounding boundary it disagrees with
any float32 pipeline.  This model instead takes the float32 planes a pipeline produced (the GPU's, or the reference
build's) and repeats that pipeline's index and scatter arithmetic on them operation by operation.  Every step is plain
float32 arithmetic except three transcendental calls:
  * WSST, Octave / Log scales: log2f of the cell's |f|;
  * synsq: atan2f of the cell.
With `libm=True` these come from the C library (glibc, through ctypes), as the reference evaluates them, and every index
is determined.  With `libm=False` they stand for the CUDA Math API's: a cell's candidates are all float32 values within
that function's documented maximum ulp error of the exact result, and an index is 'undetermined' when the candidates
lead to different rows.  `verify_columns` then checks a squeezed matrix column by column against these candidates."""
import ctypes
import ctypes.util
import itertools
import math

import numpy as np

from oracle import af_oracle as O

f32 = np.float32
TWO_PI_F = f32(2 * math.pi)             # the float the reference divides by (__vdiv_value takes a float)
PI_F = f32(3.14159265358979)             # the kernel's jump threshold
ATAN2F_ULP = 3                           # CUDA Math API, atan2f: maximum ulp error (log2f: 1, covered by two neighbours)
DROPPED = -1                             # candidate value of a cell that lands in no row

_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
for _n, _k in (("log2f", 1), ("atan2f", 2)):
    getattr(_libm, _n).restype = ctypes.c_float
    getattr(_libm, _n).argtypes = [ctypes.c_float] * _k


def glibc_log2f(x):
    x = np.asarray(x, f32)
    return np.array([_libm.log2f(float(v)) for v in x.ravel()], f32).reshape(x.shape)


def glibc_atan2f(y, x):
    y, x = np.asarray(y, f32), np.asarray(x, f32)
    return np.array([_libm.atan2f(float(a), float(b)) for a, b in zip(y.ravel(), x.ravel())], f32).reshape(y.shape)


def _c_int(v):
    return O._c_int_cast(np.asarray(v, f32))


# ---------------------------------------------------------------------------------------------------- reassignment
def reassign_index(s_h, s_dh, s_th, n, sr, hop, re_type, thresh, order=1):
    """cell indices (time, frequency) of one clip [T, W]: the oracle's float32 steps on the given planes.  Reassignment
    calls no transcendental function, so every index is determined."""
    re_f, re_t, fre, tarr = O.reassign_coords(s_h, s_dh, s_th, n, sr, hop, re_type, thresh)
    return O.reassign_indices(re_f, re_t, fre, tarr, n, order)


def _signed(s_h):
    r, i = (np.asarray(v, f32) for v in s_h)
    sign = np.where(np.arange(r.shape[-1]) % 2 == 1, f32(-1), f32(1)).astype(f32)
    return (r * sign).astype(f32), (i * sign).astype(f32)


def _amplitude(v1, v2):
    return np.sqrt(((v1 * v1).astype(f32) + (v2 * v2).astype(f32)).astype(f32)).astype(f32)


def clip_scale_exponent(s_h):
    """k_reassign_absmax + clip_scale: s = 35 - e for the clip's largest finite |re| or |im| in [2^e, 2^(e+1)), clamped
    to [-126, 126] (an all-zero or subnormal maximum has e = -127)"""
    a = np.abs(np.concatenate([np.asarray(v, f32).ravel() for v in s_h]))
    a = a[np.isfinite(a)]
    m = int(a.max().view(np.uint32)) if a.size else 0
    return int(min(126, max(-126, 35 - ((m >> 23) - 127))))


def reassign_fixed_point(s_h, ti, fi, result_type=0, start=None):
    """the GPU's output for one clip: every kept term v * 2^s rounded half to even to int64 (__float2ll_rn), summed in
    int64, converted back as (float)((double)acc * 2^-s) and added in float32 to the caller's starting planes"""
    v1, v2 = _signed(s_h)
    T, W = v1.shape
    s = clip_scale_exponent(s_h)
    scale = f32(2.0 ** s)
    ok = (ti >= 0) & (ti < T) & (fi >= 0) & (fi < W)
    dst = (np.clip(ti, 0, T - 1) * W + np.clip(fi, 0, W - 1))[ok]
    terms = [v1, v2] if result_type == 0 else [_amplitude(v1, v2)]
    start = [np.zeros((T, W), f32)] * 2 if start is None else [np.asarray(p, f32) for p in start]
    out = [p.copy() for p in start]
    for k, v in enumerate(terms):
        acc = np.zeros(T * W, np.int64)
        np.add.at(acc, dst, np.rint((v * scale).astype(f32)[ok].astype(np.float64)).astype(np.int64))
        part = (acc.astype(np.float64) * (2.0 ** -s)).astype(f32).reshape(T, W)
        out[k] = (start[k] + part).astype(f32)
    return tuple(out)


def reassign_float_sum(s_h, ti, fi, result_type=0):
    """the reference's output for one clip: float32 += into zero planes in (frame, bin) order"""
    v1, v2 = _signed(s_h)
    T, W = v1.shape
    ok = (ti >= 0) & (ti < T) & (fi >= 0) & (fi < W)
    amp = _amplitude(v1, v2)
    o_re, o_im = np.zeros((T, W), f32), np.zeros((T, W), f32)
    for i in range(T):
        m = ok[i]
        if result_type == 0:
            np.add.at(o_re, (ti[i][m], fi[i][m]), v1[i][m])
            np.add.at(o_im, (ti[i][m], fi[i][m]), v2[i][m])
        else:
            np.add.at(o_re, (ti[i][m], fi[i][m]), amp[i][m])
    return o_re, o_im


# ---------------------------------------------------------------------------------------------------- squeezing
class Index:
    """row indices of a [num, N] matrix: `idx` holds every determined cell's row (DROPPED when it lands in none);
    `cands` maps an undetermined cell (i, j) to the sorted tuple of its possible rows, or to None when any row is
    possible"""

    def __init__(self, idx, cands):
        self.idx, self.cands = idx, cands

    def columns(self):
        return sorted({j for _, j in self.cands})


def _normalise(idx, num):
    idx = np.asarray(idx, np.int64)
    return np.where((idx >= 0) & (idx < num), idx, DROPPED)


def _f32_neighbours_of_log2(a):
    """the two float32 values bracketing the exact log2 of the float32 |f| (one value where log2 is a float32)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        exact = np.log2(a.astype(np.float64))
    r = exact.astype(f32)
    lo = np.where(r.astype(np.float64) > exact, np.nextafter(r, f32(-np.inf)), r).astype(f32)
    hi = np.where(r.astype(np.float64) < exact, np.nextafter(r, f32(np.inf)), r).astype(f32)
    return lo, hi


def index_of(f, fre, sr, scale, num, log2_of=None):
    """fre_index of kernels/squeeze.cu (and the reference's index step) on float32 inst. frequencies f, with the log2f of
    |f| given (Octave / Log)"""
    f = np.asarray(f, f32)
    fre = np.asarray(fre, f32)
    fmin, fmax = f32(fre[0] / f32(sr)), f32(fre[num - 1] / f32(sr))
    with np.errstate(all="ignore"):
        if scale in (O.SCALE_OCTAVE, O.SCALE_LOG):
            l2min = f32(_libm.log2f(float(fmin)))
            l2den = f32(f32(_libm.log2f(float(fmax))) - l2min)
            v = ((((log2_of - l2min).astype(f32)) * f32(num)).astype(f32) / l2den).astype(f32)
            return _normalise(_c_int(O._roundf(v)), num)
        if scale in (O.SCALE_LINEAR, O.SCALE_LINSPACE):
            v = ((np.abs((f - fmin).astype(f32)) * f32(num)).astype(f32) / f32(fmax - fmin)).astype(f32)
            return _normalise(_c_int(O._roundf(v)), num)
    return _normalise(O.squeeze_index(f, fre, sr, scale, num), num)


def _index_with_log_candidates(f, fre, sr, scale, num, libm):
    """-> (idx, alt): equal where the index is determined"""
    if scale not in (O.SCALE_OCTAVE, O.SCALE_LOG):
        idx = index_of(f, fre, sr, scale, num)
        return idx, idx
    a = np.abs(np.asarray(f, f32))
    if libm:
        idx = index_of(f, fre, sr, scale, num, glibc_log2f(a))
        return idx, idx
    lo, hi = _f32_neighbours_of_log2(a)
    return index_of(f, fre, sr, scale, num, lo), index_of(f, fre, sr, scale, num, hi)


def wsst_inst_fre(w, dw):
    """Im(W' / W) / 2 pi in float32 operation by operation (__complexDiv, then __vdiv_value)"""
    c, d = (np.asarray(v, f32) for v in w)
    a, b = (np.asarray(v, f32) for v in dw)
    with np.errstate(all="ignore"):
        den = ((c * c).astype(f32) + (d * d).astype(f32)).astype(f32)
        im = (((b * c).astype(f32) - (a * d).astype(f32)).astype(f32) / den).astype(f32)
        return (im / TWO_PI_F).astype(f32)


def wsst_index(w, dw, fre, sr, scale, libm=False):
    """row indices of the WSST squeeze on the planes W = (re, im) and W' = (re, im), each [num, N]"""
    num = np.asarray(w[0]).shape[0]
    lo, hi = _index_with_log_candidates(wsst_inst_fre(w, dw), fre, sr, scale, num, libm)
    cands = {(int(i), int(j)): tuple(sorted({int(lo[i, j]), int(hi[i, j])})) for i, j in zip(*np.nonzero(lo != hi))}
    return Index(np.where(lo == hi, lo, DROPPED), cands)


def _phase_candidates(re, im):
    """[2 k + 1, ...] float32 values within ATAN2F_ULP ulp of the exact atan2(re, im), sorted along the first axis"""
    exact = np.arctan2(np.asarray(re, np.float64), np.asarray(im, np.float64))
    r = exact.astype(f32)
    steps = [r]
    up, dn = r, r
    for _ in range(ATAN2F_ULP + 1):
        up, dn = np.nextafter(up, f32(np.inf)), np.nextafter(dn, f32(-np.inf))
        steps += [up, dn]
    c = np.sort(np.stack(steps), axis=0)
    # keep the values whose distance to the exact result is at most ATAN2F_ULP ulp of that result (the ulp of the
    # nearest float32); an extra step was generated so the boundary is decided by this test, not by the loop count
    ulp = np.abs(np.nextafter(r, f32(np.inf)).astype(np.float64) - r.astype(np.float64))
    keep = np.abs(c.astype(np.float64) - exact[None]) <= ATAN2F_ULP * ulp[None]
    lo = np.where(keep, c, np.inf).min(axis=0).astype(f32)
    hi = np.where(keep, c, -np.inf).max(axis=0).astype(f32)
    return lo, hi


def _jump(dlt):
    return np.where(dlt > PI_F, -1, np.where(dlt < -PI_F, 1, 0))


def _unwrapped(ph, K):
    return (np.asarray(ph, f32).astype(np.float64) + 6.283185307179586 * np.asarray(K, np.float64)).astype(f32)


def synsq_index(re, im, fre, sr, scale, libm=False):
    """row indices of the synsq squeeze of the planes (re, im) [num, N]: phase atan2f(re, im), the kernel's unwrap (a
    running count K of +-1 jumps where the raw difference leaves [-pi, pi], u = fl(p + 2 pi K)), first difference
    (0 in column 0, column N-1 repeats column N-2), / 2 pi, index.

    With libm=False every phase is an interval [lo, hi] of float32 candidates.  A jump decision is determined when the
    smallest and the largest candidate difference agree (float subtraction is monotone); after an undetermined jump the
    rest of the row is open (any row).  A difference's interval follows from the intervals of u; the index is determined
    when both ends give the same row and the interval crosses no point where the index stops being monotone (0, and
    +-fmin on the linear scales)."""
    re, im = np.asarray(re, f32), np.asarray(im, f32)
    num, n = re.shape
    if libm:
        lo = hi = glibc_atan2f(re, im)
    else:
        lo, hi = _phase_candidates(re, im)
    with np.errstate(all="ignore"):
        dmin = np.zeros_like(lo)
        dmax = np.zeros_like(lo)
        dmin[:, 1:] = (lo[:, 1:] - hi[:, :-1]).astype(f32)
        dmax[:, 1:] = (hi[:, 1:] - lo[:, :-1]).astype(f32)
    jmin, jmax = _jump(dmax), _jump(dmin)                  # larger difference -> smaller jump
    undetermined_jump = jmin != jmax
    first_open = np.where(undetermined_jump.any(axis=1), undetermined_jump.argmax(axis=1), n)
    K = np.cumsum(jmin, axis=1)                             # valid before each row's first undetermined jump
    u_lo, u_hi = _unwrapped(lo, K), _unwrapped(hi, K)
    with np.errstate(all="ignore"):
        f_lo = np.zeros_like(lo)
        f_hi = np.zeros_like(lo)
        f_lo[:, 1:] = ((u_lo[:, 1:] - u_hi[:, :-1]).astype(f32) / TWO_PI_F).astype(f32)
        f_hi[:, 1:] = ((u_hi[:, 1:] - u_lo[:, :-1]).astype(f32) / TWO_PI_F).astype(f32)
    f_lo[:, n - 1], f_hi[:, n - 1] = f_lo[:, n - 2], f_hi[:, n - 2]
    a_lo, a_hi = _index_with_log_candidates(f_lo, fre, sr, scale, num, libm)
    b_lo, b_hi = _index_with_log_candidates(f_hi, fre, sr, scale, num, libm)
    fmin = f32(np.asarray(fre, f32)[0] / f32(sr))
    cross = (f_lo <= 0) & (f_hi >= 0)
    if scale in (O.SCALE_LINEAR, O.SCALE_LINSPACE):
        cross |= ((f_lo <= fmin) & (f_hi >= fmin)) | ((f_lo <= -fmin) & (f_hi >= -fmin))
    same = (a_lo == a_hi) & (a_lo == b_lo) & (b_lo == b_hi) & ~(cross & (f_lo != f_hi))
    cols = np.arange(n)[None, :]
    # the open part of a row: from the column of its first undetermined jump on (the last column follows column N-2)
    open_ = cols >= first_open[:, None]
    open_[:, n - 1] = open_[:, n - 2]
    idx = np.where(same & ~open_, a_lo, DROPPED)
    cands = {}
    for i, j in zip(*np.nonzero(open_)):
        cands[(int(i), int(j))] = None
    for i, j in zip(*np.nonzero(~same & ~open_)):
        rows = _enumerate_synsq_cell(lo, hi, K, int(i), int(j), n, fre, sr, scale, num)
        if len(rows) == 1:
            idx[i, j] = rows[0]
        else:
            cands[(int(i), int(j))] = rows
    return Index(idx, cands)


def _enumerate_synsq_cell(lo, hi, K, i, j, n, fre, sr, scale, num):
    """all rows an undetermined synsq cell can reach: every candidate pair (u, u_prev) of its difference"""
    jj = n - 2 if j == n - 1 else j

    def values(a, b):
        out = [a]
        while out[-1] < b:
            out.append(np.nextafter(out[-1], f32(np.inf)))
        return np.array(out, f32)

    cur = _unwrapped(values(lo[i, jj], hi[i, jj]), K[i, jj])
    prev = _unwrapped(values(lo[i, jj - 1], hi[i, jj - 1]), K[i, jj - 1])
    with np.errstate(all="ignore"):
        f = ((cur[:, None] - prev[None, :]).astype(f32) / TWO_PI_F).astype(f32).ravel()
    rows = set()
    for half in _index_with_log_candidates(f, fre, sr, scale, num, False):
        rows.update(int(v) for v in half)
    return tuple(sorted(rows))


def scatter(w, idx, thresh, start=None):
    """out[idx[i, j], j] += W[i, j] for rows i ascending where idx is a row and fl(fl(re^2) + fl(im^2)) > fl(thresh^2);
    float32 additions starting from the caller's planes"""
    re, im = (np.asarray(v, f32) for v in w)
    num, n = re.shape
    t2 = f32(f32(thresh) * f32(thresh))
    out = [np.zeros((num, n), f32), np.zeros((num, n), f32)] if start is None else [np.array(p, f32) for p in start]
    cols = np.arange(n)
    keep = (idx >= 0) & (power(re, im) > t2)
    for i in range(num):
        ok = keep[i]
        r = idx[i][ok]
        out[0][r, cols[ok]] += re[i][ok]
        out[1][r, cols[ok]] += im[i][ok]
    return tuple(out)


def power(re, im):
    re, im = np.asarray(re, f32), np.asarray(im, f32)
    return ((re * re).astype(f32) + (im * im).astype(f32)).astype(f32)


def _scatter_column(re, im, rows, kept, start_re, start_im):
    o_re, o_im = start_re.copy(), start_im.copy()
    for i in range(re.shape[0]):
        r = rows[i]
        if r >= 0 and kept[i]:
            o_re[r] = f32(o_re[r] + re[i])
            o_im[r] = f32(o_im[r] + im[i])
    return o_re, o_im


def verify_columns(got, w, index, thresh, start=None, max_assignments=64):
    """check a squeezed matrix `got` = (re, im) against the planes w = (re, im) and an Index:
      * a column whose cells are all determined must match bit for bit;
      * a column with at most 3 undetermined cells, each with a finite candidate set, and at most `max_assignments`
        assignments must equal, bit for bit, the column of one of those assignments;
      * any other column: per row, |got - determined part| <= sum of |W| of the undetermined cells that can land there,
        plus the float32 rounding of that row's sum.
    Cells below the threshold are dropped whatever their index and never count as undetermined.
    -> dict with the failing columns and the shares of undetermined cells / columns"""
    re, im = (np.asarray(v, f32) for v in w)
    num, n = re.shape
    start = (np.zeros((num, n), f32), np.zeros((num, n), f32)) if start is None else tuple(np.asarray(p, f32) for p in start)
    t2 = f32(f32(thresh) * f32(thresh))
    kept = power(re, im) > t2
    g_re, g_im = (np.asarray(v, f32) for v in got)
    # a cell below the threshold lands nowhere, whatever its index
    index = Index(index.idx, {k: c for k, c in index.cands.items() if kept[k]})
    # determined part: undetermined cells left out
    det_idx = index.idx.copy()
    for (i, j) in index.cands:
        det_idx[i, j] = DROPPED
    d_re, d_im = scatter((re, im), det_idx, thresh, start)
    by_col = {}
    for (i, j), c in index.cands.items():
        by_col.setdefault(j, []).append((i, c))
    bad_det = ~((g_re.view(np.uint32) == d_re.view(np.uint32)) & (g_im.view(np.uint32) == d_im.view(np.uint32))).all(axis=0)
    for j in by_col:
        bad_det[j] = False
    failures = [int(j) for j in np.nonzero(bad_det)[0]]
    enumerated = bounded = 0
    for j, cells in by_col.items():
        cands = [c for _, c in cells]
        if len(cells) <= 3 and all(c is not None for c in cands) and math.prod(len(c) for c in cands) <= max_assignments:
            enumerated += 1
            rows = index.idx[:, j].copy()
            ok = False
            for choice in itertools.product(*cands):
                for (i, _), r in zip(cells, choice):
                    rows[i] = r
                o_re, o_im = _scatter_column(re[:, j], im[:, j], rows, kept[:, j], start[0][:, j], start[1][:, j])
                if np.array_equal(o_re.view(np.uint32), g_re[:, j].view(np.uint32)) and \
                        np.array_equal(o_im.view(np.uint32), g_im[:, j].view(np.uint32)):
                    ok = True
                    break
            if not ok:
                failures.append(int(j))
            continue
        bounded += 1
        b_re, b_im = np.zeros(num), np.zeros(num)
        for i, c in cells:
            if not kept[i, j]:
                continue
            targets = range(num) if c is None else [r for r in c if r >= 0]
            for r in targets:
                b_re[r] += abs(float(re[i, j]))
                b_im[r] += abs(float(im[i, j]))
        col_rows = np.where(kept[:, j], index.idx[:, j], DROPPED)
        terms = np.bincount(col_rows[col_rows >= 0], minlength=num)[:num] + len(cells)
        mag_re = np.abs(start[0][:, j]).astype(np.float64) + b_re
        mag_im = np.abs(start[1][:, j]).astype(np.float64) + b_im
        for r in np.nonzero(col_rows >= 0)[0]:
            mag_re[col_rows[r]] += abs(float(re[r, j]))
            mag_im[col_rows[r]] += abs(float(im[r, j]))
        slack_re = (terms + 1) * 2.0 ** -23 * mag_re
        slack_im = (terms + 1) * 2.0 ** -23 * mag_im
        e_re = np.abs(g_re[:, j].astype(np.float64) - d_re[:, j])
        e_im = np.abs(g_im[:, j].astype(np.float64) - d_im[:, j])
        if not ((e_re <= b_re + slack_re).all() and (e_im <= b_im + slack_im).all()):
            failures.append(int(j))
    return {"failures": sorted(failures), "undetermined_cells": len(index.cands), "cells": num * n,
            "undetermined_columns": len(by_col) / n, "enumerated_columns": enumerated, "bounded_columns": bounded}


def crafted_threshold_pairs(count=8, thresh=0.001, seed=0):
    """float32 pairs (v1, v2) whose |W|^2 test against fl(thresh^2) comes out one way evaluated operation by operation,
    fl(fl(v1^2) + fl(v2^2)), and the other way with either FMA contraction, fma(v2, v2, fl(v1^2)) or
    fma(v1, v1, fl(v2^2)).  -> (v1, v2, kept by the op-by-op test).  The float64 evaluation here is exact (float32
    squares and their sums fit in 53 bits); tests re-check it with fractions."""
    t2 = float(f32(f32(thresh) * f32(thresh)))
    rng = np.random.default_rng(seed)
    v1s, v2s, kept = [], [], []
    for _ in range(100 * count):
        if len(v1s) >= count:
            break
        v2 = f32(rng.uniform(0.3, 0.7) * thresh)
        v1c = f32(math.sqrt(max(t2 - float(v2) ** 2, 0.0)))
        v1 = v1c + (np.arange(-64, 65) * np.spacing(v1c)).astype(f32)
        a, b = v1.astype(np.float64) ** 2, float(v2) ** 2
        fa, fb = a.astype(f32).astype(np.float64), float(f32(b))
        op = (fa + fb).astype(f32).astype(np.float64) > t2
        fma2 = (b + fa).astype(f32).astype(np.float64) > t2
        fma1 = (a + fb).astype(f32).astype(np.float64) > t2
        for k in np.nonzero((op != fma1) & (op != fma2))[0][:1]:
            v1s.append(v1[k]); v2s.append(v2); kept.append(bool(op[k]))
    assert len(v1s) == count, "no crafted threshold pairs found"
    return np.array(v1s, f32), np.array(v2s, f32), np.array(kept)
