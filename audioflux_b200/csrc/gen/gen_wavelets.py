#!/usr/bin/env python3
"""Generate kernels/wavelet_coef_gen.h: the decomposition filters (loD, hiD) of the discrete wavelet transforms, built from
their mathematical definitions and rounded to 6 decimals.

    python3 gen/gen_wavelets.py kernels/wavelet_coef_gen.h      (needs mpmath; run from audioflux_b200/csrc)

Conventions (those of DWTObj's filters): h is the synthesis lowpass of sum sqrt(2); loD = h reversed and
hiD[n] = (-1)^(n+1) h[n].

- Daubechies dbN (haar = db1): the maximally flat half-band product P(y) = sum_{k<N} C(N-1+k, k) y^k with
  y = (2 - z - 1/z)/4.  Each root y of P gives the pair z, 1/z of z^2 - (2 - 4y) z + 1; h = (1 + z)^N times the
  roots inside the unit circle (minimum phase).  The roots are found with mpmath at 120 digits: at N = 30 the
  binomial coefficients reach 1e17 and float64 roots lose the 6th decimal.
- Symlets symN: the same roots; of each root group (a real root, or a conjugate pair) either the inside or the outside
  member.  symN = dbN for N < 4.  For N >= 4 the selection is the one whose frequency response has the most linear
  phase: the least squared deviation of the unwrapped phase from its least-squares line over 512 points of
  [0, 0.78 pi].  That criterion cannot tell a filter from its time reverse; of the two, the one whose loD peaks first.
- Biorthogonal spline wavelets biorNr.Nd: h = sqrt(2) ((1 + z)/2)^Nr (a B-spline) and the analysis lowpass
  h~ = sqrt(2) ((1 + z)/2)^Nd P_l(y), l = (Nr + Nd)/2, with P_l the Daubechies product above.  Both are centred in a
  common even length L: even-length filters start at (L - len)/2; of odd length, loD (= h~, symmetric) is centred on
  L/2 and the synthesis lowpass h that hiD modulates on L/2 - 1.  hiD[n] = (-1)^(n+1) h[n].

tests/test_wavelet_cpu.py checks that every filter in the table reproduces DWTObj's reference table to every printed
decimal; only the orders that do are listed (DB_ORDERS, SYM_ORDERS, BIOR_ORDERS).  Refused, with the reason recorded in
REFUSED:
- db40: the reference table differs from the construction by 1e-6 in 9 taps (its table sums to 1.414211, not
  sqrt(2) = 1.414214, beyond the 6-decimal rounding);
- sym7, sym10, sym20, sym30: the phase-linearity selection above picks another root selection than the reference's;
- coif1-5: the moment equations have several solutions and no selection rule has been found that picks the
  reference's;
- bior4.4, bior5.5, bior6.8: not spline wavelets (their factorisation splits the roots of P_l between the two sides);
- fk4-22 and dmey: optimised or fitted filters, with no construction to regenerate them from.
"""
import itertools
import sys

import mpmath as mp
import numpy as np

mp.mp.dps = 120

# WaveletDiscreteType (afb200_dwt.h)
HAAR, DB, SYM, COIF, FK, BIOR, DMEY = range(7)

DB_ORDERS = (2, 3, 4, 5, 6, 7, 8, 9, 10, 20, 30)
SYM_ORDERS = (2, 3, 4, 5, 6, 8, 9)
BIOR_ORDERS = ((1, 1), (1, 3), (1, 5), (2, 2), (2, 4), (2, 6), (2, 8), (3, 1), (3, 3), (3, 5), (3, 7), (3, 9))
REFUSED = {
    (DB, 40, 0): "the reference table differs from the construction by 1e-6 in 9 taps",
    **{(SYM, n, 0): "the most-linear-phase root selection differs from the reference's" for n in (7, 10, 20, 30)},
    **{(COIF, n, 0): "no construction reproduces the reference's coiflet table" for n in (1, 2, 3, 4, 5)},
    **{(BIOR, a, b): "not a spline wavelet; no construction reproduces the reference's table"
       for a, b in ((4, 4), (5, 5), (6, 8))},
    **{(FK, n, 0): "an optimised filter with no construction to regenerate it from" for n in (4, 6, 8, 14, 18, 22)},
    (DMEY, 0, 0): "a fitted FIR with no construction to regenerate it from",
}


def _yroots(n):
    if n == 1:
        return []
    c = [mp.binomial(n - 1 + k, k) for k in range(n)]
    return mp.polyroots(c[::-1], maxsteps=2000, extraprec=2000)


def _inside(y):
    b = 2 - 4 * y
    z = (b + mp.sqrt(b * b - 4)) / 2
    return z if abs(z) < 1 else 1 / z


def _poly(roots):
    p = [mp.mpc(1)]
    for r in roots:
        q = [mp.mpc(0)] * (len(p) + 1)
        for i, a in enumerate(p):
            q[i] += a
            q[i + 1] -= a * r
        p = q
    return np.array([float(mp.re(a)) for a in p])


def _scaled(p):
    return p * np.sqrt(2) / p.sum()


def _from_h(h):
    return h[::-1].copy(), np.array([(-1) ** (n + 1) * h[n] for n in range(len(h))])


def daubechies(n):
    return _from_h(_scaled(_poly([_inside(y) for y in _yroots(n)] + [-1] * n)))


def _groups(n):
    ys = list(_yroots(n))
    out = []
    while ys:
        y = ys.pop(0)
        if abs(mp.im(y)) < mp.mpf(10) ** -60:
            out.append([_inside(y)])
        else:
            j = min(range(len(ys)), key=lambda k: abs(ys[k] - mp.conj(y)))
            ys.pop(j)
            z = _inside(y)
            out.append([z, mp.conj(z)])
    return out


def _phase_dev(h, wmax=0.78 * np.pi, nw=512):
    w = np.linspace(0, wmax, nw)
    ph = np.unwrap(np.angle(np.exp(-1j * np.outer(w, np.arange(len(h)))) @ h))
    a = np.vstack([w, np.ones_like(w)]).T
    c, *_ = np.linalg.lstsq(a, ph, rcond=None)
    return float(np.sum((ph - a @ c) ** 2))


def symlet(n):
    if n < 4:
        return daubechies(n)
    gs = _groups(n)
    cands = []
    for bits in itertools.product((0, 1), repeat=len(gs)):
        zs = [z if b == 0 else 1 / z for b, g in zip(bits, gs) for z in g]
        h = _scaled(_poly(zs + [-1] * n))
        lo, hi = _from_h(h)
        cands.append((round(_phase_dev(h), 9), int(np.argmax(np.abs(lo))), lo, hi))
    cands.sort(key=lambda c: (c[0], c[1]))
    return cands[0][2], cands[0][3]


def _centre(f, length, odd_centre):
    out = np.zeros(length)
    s = (length - len(f)) // 2 if len(f) % 2 == 0 else odd_centre - (len(f) - 1) // 2
    out[s:s + len(f)] = f
    return out


def bior_spline(nr, nd):
    l = (nr + nd) // 2
    y = np.array([-0.25, 0.5, -0.25])          # y = (2 - z - 1/z)/4 as a Laurent polynomial
    pl, yk = np.zeros(2 * l - 1), np.array([1.0])
    for k in range(l):                          # P_l(y), centred: y^k spans 2k+1 taps
        pl[l - 1 - k:l + k] += float(mp.binomial(l - 1 + k, k)) * yk
        yk = np.convolve(yk, y)
    ht = _scaled(np.convolve(_binom(nd), pl))
    h = _scaled(_binom(nr))
    length = max(len(ht), len(h))
    length += length % 2
    lo = _centre(ht, length, length // 2 - 1)
    hr = _centre(h, length, length // 2 - 1)
    return lo[::-1].copy(), np.array([(-1) ** (n + 1) * hr[n] for n in range(length)])


def _binom(n):
    return np.array([float(mp.binomial(n, k)) for k in range(n + 1)])


def table():
    """{(type, t1, t2): (loD, hiD)} of every supported combination, rounded to 6 decimals (t2 = 0 unless Bior)"""
    t = {(HAAR, 0, 0): daubechies(1)}
    t.update({(DB, n, 0): daubechies(n) for n in DB_ORDERS})
    t.update({(SYM, n, 0): symlet(n) for n in SYM_ORDERS})
    t.update({(BIOR, a, b): bior_spline(a, b) for a, b in BIOR_ORDERS})
    return {k: (np.round(lo, 6) + 0.0, np.round(hi, 6) + 0.0) for k, (lo, hi) in t.items()}


def emit(path):
    t = table()
    lines = ["/* Generated by gen/gen_wavelets.py -- do not edit.  Decomposition filters of the discrete wavelet",
             " * transforms, built from their definitions and rounded to 6 decimals. */",
             "#ifndef WAVELET_COEF_GEN_H", "#define WAVELET_COEF_GEN_H", "",
             "typedef struct { int type, t1, t2, length; const float *lo, *hi; } AfWaveletCoef;", ""]
    names = []
    for (ty, a, b), (lo, hi) in t.items():
        name = f"af_w{ty}_{a}_{b}"
        names.append((ty, a, b, len(lo), name))
        for suffix, arr in (("lo", lo), ("hi", hi)):
            vals = ", ".join(f"{v:.6f}f" for v in arr)
            lines.append(f"static const float {name}_{suffix}[{len(arr)}] = {{{vals}}};")
    lines += ["", "static const AfWaveletCoef af_wavelet_coefs[] = {"]
    lines += [f"    {{{ty}, {a}, {b}, {n}, {name}_lo, {name}_hi}}," for ty, a, b, n, name in names]
    lines += ["};", "", "typedef struct { int type, t1, t2; const char *why; } AfWaveletRefusal;", "",
              "static const AfWaveletRefusal af_wavelet_refusals[] = {"]
    lines += [f'    {{{ty}, {a}, {b}, "{why}"}},' for (ty, a, b), why in REFUSED.items()]
    lines += ["};", "", "#endif", ""]
    with open(path, "w") as f:
        f.write("\n".join(lines))


if __name__ == "__main__":
    emit(sys.argv[1] if len(sys.argv) > 1 else "kernels/wavelet_coef_gen.h")
