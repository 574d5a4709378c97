"""Float64 numpy restatement of the reference's NCF and cepstrum pitch trackers (PitchNCF, PitchCEP) with error bounds,
the case lists, and ctypes drivers that work on either library.

src/mir/_pitch_ncf.c and src/mir/_pitch_cep.c, with n = 2^radix2Exp:
  - new (:77-164 / :77-166): samplate outside (0, 196000] -> 32000; lowFre < 27 -> 32; highFre not in (lowFre,
    samplate/2) (integer samplate/2) -> lowFre 32, highFre 2000; radix2Exp outside 1 .. 30 -> 12; slideLength <= 0 ->
    n/4; minIndex = roundf(samplate/highFre), maxIndex = roundf(samplate/lowFre) (float quotients); NCF takes any
    window (Rect by default), CEP only windows up to Hamm (Hamm otherwise);
  - NCF per frame (:380-494): r = the autocorrelation of the windowed frame (2n-point FFT, |X|^2, inverse), slot j holds
    r[j+1] / sqrt(r[0]) for j = minIndex-1 .. maxIndex-1 and slot maxIndex holds 0; __vmax's first maximum over slots
    minIndex .. maxIndex; fre = samplate / (slot + 1);
  - CEP per frame (:381-474): c = IFFT_2n(log |FFT_2n(x)|^2); __vmax's first maximum over c[minIndex .. maxIndex];
    fre = samplate / (index + 1).
A NaN first slot stays __vmax's maximum: a frame whose windowed samples are all zero, or that holds a NaN, gives
samplate / (minIndex + 1).

Error bounds.  A float32 radix-2 FFT of N <= 2^15 points has an l2 error of about 2^-24 log2 N <= 9e-7 of its output's
norm, a bound on every entry.  NCF: the correlation runs a forward transform, the power and an inverse, so every lag is
within KAPPA ||frame||^2 = KAPPA r[0] of the float64 value (KAPPA = 4e-6, as the PEF and YIN oracles), and every slot
within KAPPA sqrt(r[0]) after the normalisation; the 0 slot is exact.  CEP: every bin is within DELTA = KAPPA / 2
sqrt(2n) ||frame|| of |X_k|, so log |X_k|^2 lies in [2 log(|X_k| - DELTA), 2 log(|X_k| + DELTA)] (unbounded below once
|X_k| <= DELTA), widened by the float32 rounding of the power and the log; the cepstrum interval's radius is the mean of
those radii plus KAPPA times the l2 norm of the log spectrum over sqrt(2n), the inverse transform's own error.  A slot
whose interval reaches the top slot's is a candidate; the frame's arg-max is undetermined when there are several."""
import numpy as np

from _pitch_c import c_free, c_new, c_pitch, signal, time_length
from oracle import af_oracle as O

W_RECT, W_HANN, W_HAMM, W_BLACKMAN, W_KAISER = O.W_RECT, O.W_HANN, O.W_HAMM, O.W_BLACKMAN, O.W_KAISER
f32 = np.float32
KAPPA = 4e-6
U = 2.0 ** -24
KINDS = ("ncf", "cep")


def params(kind, sr=None, lf=None, hf=None, r2=None, slide=None, wt=None):
    """new -> dict; status 0, or this library's refusals -2 (radix2Exp > 14) and -3 (NCF maxIndex >= n or minIndex < 1,
    CEP maxIndex > 2n - 1, an empty lag range)"""
    sr = sr if sr is not None and 0 < sr <= 196000 else 32000
    low = f32(lf) if lf is not None and f32(lf) >= 27 else f32(32)
    high = f32(2000)
    if hf is not None:
        if f32(hf) > low and f32(hf) < f32(sr // 2):
            high = f32(hf)
        else:
            low, high = f32(32), f32(2000)
    r2 = r2 if r2 is not None and 1 <= r2 <= 30 else 12
    n = 1 << r2
    hop = slide if slide is not None and slide > 0 else max(1, n // 4)
    if kind == "ncf":
        win = W_RECT if wt is None else wt
    else:
        win = wt if wt is not None and wt <= W_HAMM else W_HAMM
    # roundf of the float quotients: halves away from zero (both are positive), in double so that + 0.5 is exact
    mi, ma = int(np.floor(float(f32(sr) / high) + 0.5)), int(np.floor(float(f32(sr) / low) + 0.5))
    p = dict(kind=kind, sr=sr, n=n, r2=r2, slide=hop, low=low, high=high, wt=win, min_index=mi, max_index=ma)
    if r2 > 14:
        return dict(p, status=-2)
    if kind == "ncf" and (ma >= n or mi < 1):
        return dict(p, status=-3)
    if kind == "cep" and ma > 2 * n - 1:
        return dict(p, status=-3)
    if ma < mi:
        return dict(p, status=-3)
    return dict(p, status=0)


def _frames(x, p):
    n, hop = p["n"], p["slide"]
    T = time_length(len(x), n, hop)
    idx = np.arange(T)[:, None] * hop + np.arange(n)[None, :]
    return (np.asarray(x, f32)[idx] * O.fft_window(p["wt"], n)[None, :]).astype(np.float64)     # float32 products


def _slots_ncf(xw, p):
    """the slot values minIndex .. maxIndex, their error radii, and the frames decided by their first slot"""
    n, lo, hi = p["n"], p["min_index"], p["max_index"]
    with np.errstate(invalid="ignore"):
        r = np.fft.irfft(np.abs(np.fft.rfft(xw, 2 * n, axis=1)) ** 2, 2 * n, axis=1)
    r0 = np.sum(xw * xw, axis=1)
    first = ~np.isfinite(r0) | (r0 == 0)
    rms = np.sqrt(np.where(first, 1.0, r0))
    v = np.zeros((xw.shape[0], hi - lo + 1))
    v[:, :hi - lo] = r[:, lo + 1:hi + 1] / rms[:, None]
    rad = np.full(v.shape, KAPPA) * rms[:, None]
    rad[:, -1] = 0.0
    return v, rad, first


def _slots_cep(xw, p):
    n, lo, hi = p["n"], p["min_index"], p["max_index"]
    N = 2 * n
    norm = np.sqrt(np.sum(xw * xw, axis=1))
    first = ~np.isfinite(norm) | (norm == 0)
    xw = np.where(first[:, None], 1.0, xw)
    mag = np.abs(np.fft.rfft(xw, N, axis=1))                           # bins 0 .. n
    delta = (KAPPA / 2) * np.sqrt(N) * norm[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        L = 2 * np.log(mag)
        lo_l = 2 * np.log(np.maximum(mag - delta, 0.0))
        hi_l = 2 * np.log(mag + delta)
        rho = np.maximum(L - lo_l, hi_l - L) + 4 * U * (np.abs(L) + 1)  # the power's and the log's float32 rounding
    rho = np.where(np.isnan(rho), np.inf, rho)
    full = np.concatenate([L, L[:, n - 1:0:-1]], axis=1)                # the 2n bins, Hermitian
    rho_full = np.concatenate([rho, rho[:, n - 1:0:-1]], axis=1)
    with np.errstate(invalid="ignore"):
        c = np.fft.irfft(np.where(np.isfinite(L), L, 0.0), N, axis=1)
    rad = np.mean(rho_full, axis=1) + KAPPA * np.sqrt(np.sum(np.where(np.isfinite(full), full, 0.0) ** 2, axis=1) / N)
    rad = np.where(np.isfinite(rad), rad, np.inf)
    v = c[:, lo:hi + 1]
    return v, np.broadcast_to(rad[:, None], v.shape), first


def pitch(x, p, block=64):
    """one clip -> (frequencies [T] float32, candidate indices per frame as sets)"""
    n, hop, lo = p["n"], p["slide"], p["min_index"]
    slots = _slots_ncf if p["kind"] == "ncf" else _slots_cep
    best, cands = [], []
    for t0 in range(0, time_length(len(x), n, hop), block):
        v, rad, first = slots(_frames(x[t0 * hop:(t0 + block - 1) * hop + n], p), p)
        for t in range(v.shape[0]):
            if first[t]:
                best.append(lo)
                cands.append({lo})
                continue
            if not np.isfinite(rad[t]).all():
                best.append(lo + int(np.argmax(v[t])))
                cands.append(set(range(lo, p["max_index"] + 1)))
                continue
            k = int(np.argmax(v[t]))
            floor = np.max(v[t] - rad[t])
            best.append(lo + k)
            cands.append({lo + int(i) for i in np.flatnonzero(v[t] + rad[t] >= floor)})
    return fre(np.array(best, int), p), cands


def fre(index, p):
    """samplate / (index + 1) in double, stored as float"""
    return (p["sr"] / (np.asarray(index, np.float64) + 1)).astype(f32)


def agree(got, want, cands, p):
    """(ok, frames decided by a candidate): each frame's frequency is exactly the oracle's, or exactly the frequency of
    one of its candidate indices"""
    got = np.asarray(got)
    if got.shape != want.shape:
        return False, []
    alt = []
    for t in np.flatnonzero(got != want):
        if got[t] not in set(fre(sorted(cands[t]), p).tolist()):
            return False, [int(t)]
        alt.append(int(t))
    return True, alt


# ---- cases ----

def cases(kind):
    """[(name, dict(ctor=dict(...), length, kind))]: ctor arguments left out are passed as NULL"""
    out = []

    def add(name, length, sig="tones", **ctor):
        out.append((name, dict(ctor=ctor, length=length, kind=sig)))

    add("default", 4096 + 30 * 1024)
    add("default_null", 4096 + 20 * 1024, slide=None)
    for r2, sr in ((9, 8000), (10, 11025), (11, 16000), (13, 44100), (14, 96000)):
        n = 1 << r2
        add(f"r{r2}_sr{sr}", n + 20 * (n // 4), sr=sr, r2=r2, slide=n // 4)
    for sr in (22050, 48000):
        add(f"sr{sr}", 2 * sr, sr=sr, r2=12, slide=1000)
    for w in ((W_RECT, W_HANN, W_HAMM, W_BLACKMAN, W_KAISER) if kind == "ncf" else (W_RECT, W_HANN, W_HAMM, W_BLACKMAN)):
        add(f"win{w}", 32000, wt=w, r2=12, slide=1024)
    add("slide_gt_n", 60000, r2=12, slide=5000)
    add("slide1", 2048 + 40, r2=11, slide=1, sig="noise")
    add("lf_fallback", 32000, lf=20.0, hf=1000.0, r2=12, slide=1024)
    add("hf_fallback", 32000, sr=8000, lf=100.0, hf=4500.0, r2=12, slide=1024)
    add("sr_fallback", 32000, sr=0, r2=12, slide=1024)
    add("narrow", 32000, lf=150.0, hf=400.0, r2=12, slide=1024)
    add("one_lag", 32000, lf=1000.0, hf=1001.0, r2=12, slide=1024)
    for sig in ("silence", "dc", "alt", "noise", "low", "chirp", "gaps", "nan"):       # sig_chirp: the glide
        add(f"sig_{sig}", 48000, sig="glide" if sig == "chirp" else sig, sr=32000, r2=12, slide=1024)
    add("sig_chirp_r13", 8192 + 30 * 2048, sig="glide", sr=44100, r2=13, slide=2048)
    add("sentinel", 32000, sig="tone4638", sr=32000, lf=900.0, hf=1000.0, r2=12, slide=1024)
    add("r5", 600, sr=8000, lf=300.0, hf=1000.0, r2=5, slide=16, sig="noise")
    return out


def case_params(kind, kw):
    return params(kind, **kw["ctor"])


def case_signal(kind, name, kw):
    return signal(kw["kind"], kw["length"], case_params(kind, kw)["sr"], sum(map(ord, name)))


def oracle_case(kind, name, kw):
    return pitch(case_signal(kind, name, kw), case_params(kind, kw))


def c_case(lib, kind, name, kw):
    st, obj = c_new(lib, kind, **kw["ctor"])
    assert st == 0, (kind, name, st)
    out = c_pitch(lib, kind, obj, case_signal(kind, name, kw))
    c_free(lib, kind, obj)
    return out
