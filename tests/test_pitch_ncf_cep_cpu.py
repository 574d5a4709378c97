"""PitchNCF and PitchCEP without a GPU: the float64 oracle against the reference build (or its stored outputs in
tests/golden/pitch_ncf_cep.npz) over frame sizes, samplates, windows, slides and signals (silence, NaN, alternating
signs, a constant, the NCF 0 slot); the statuses of new and calTimeLength against the reference, streaming included; the
refusals (which need no device); the exported and bound symbols of include/afb200_pitch_{ncf,cep}.h and afb200_ext.h;
and the Python classes' arguments.

Run as a script, it rewrites tests/golden/pitch_ncf_cep.npz from the reference build (oracle/_ref):

    python tests/test_pitch_ncf_cep_cpu.py"""
import numpy as np
import pytest

from _parity_kit import GoldenStore, check_symbols, ref_lib_or_none      # first: conftest puts the root on sys.path
import _pitch_c as PC
import _pitch_ncf_cep_oracle as PO

CASES = {k: dict(PO.cases(k)) for k in PO.KINDS}
ALL = [(k, name) for k in PO.KINDS for name in CASES[k]]


def _live(keys):
    lib = ref_lib_or_none()
    out = {}
    for key in keys:
        kind, name = key.split("/")
        out[key] = PO.c_case(lib, kind, name, CASES[kind][name])
    return out


GOLD = GoldenStore("pitch_ncf_cep.npz", _live, lambda: {f"{k}/{n}" for k, n in ALL})


@pytest.mark.parametrize("kind,name", ALL)
def test_oracle_matches_reference(kind, name):
    kw = CASES[kind][name]
    p = PO.case_params(kind, kw)
    assert p["status"] == 0
    got = GOLD.outputs({f"{kind}/{name}"})[f"{kind}/{name}"]
    want, cands = PO.oracle_case(kind, name, kw)
    ok, alt = PO.agree(got, want, cands, p)
    assert ok, (kind, name, alt, got[alt], want[alt])
    if kw["kind"] not in ("dc", "alt"):            # exact zeros in the spectrum: every cepstrum slot is a candidate
        assert len(alt) <= max(2, len(want) // 10), (kind, name, alt)


def test_cases_cover_the_edges():
    """n = 2^9 .. 2^14, samplates 8 kHz .. 96 kHz, slides above n, the single-slot range, and the NCF 0 slot winning
    (32000 / 37) for a 32000/69 Hz tone between 900 and 1000 Hz; silence and the NaN sample give samplate /
    (minIndex + 1), alternating signs 32000 / 18 for NCF"""
    for kind in PO.KINDS:
        ps = {k: PO.case_params(kind, kw) for k, kw in CASES[kind].items()}
        assert {p["n"] for p in ps.values()} >= {1 << r for r in range(9, 15)}
        assert min(p["sr"] for p in ps.values()) == 8000 and max(p["sr"] for p in ps.values()) == 96000
        assert ps["slide_gt_n"]["slide"] > ps["slide_gt_n"]["n"]
        assert ps["one_lag"]["min_index"] == ps["one_lag"]["max_index"]
        for sig in ("sig_silence", "sig_nan"):
            want, cands = PO.oracle_case(kind, sig, CASES[kind][sig])
            if sig == "sig_silence":
                assert (want == np.float32(32000 / 17)).all()
            else:
                for t in range(20, 24):                                          # the frames holding the NaN
                    assert cands[t] == {16} and want[t] == np.float32(32000 / 17)
    want, cands = PO.oracle_case("ncf", "sentinel", CASES["ncf"]["sentinel"])
    assert (want == np.float32(32000 / 37)).all() and all(c == {36} for c in cands)
    want, _ = PO.oracle_case("ncf", "sig_alt", CASES["ncf"]["sig_alt"])
    assert (want == np.float32(32000 / 18)).all()


def test_golden_file_matches_reference_build():
    GOLD.check_file()


def _grid():
    grid = []
    for sr in (None, -1, 900, 8000, 11025, 32000, 44100, 196001):
        for lf in (None, 20.0, 27.0, 100.0, 3000.0):
            for hf in (None, 90.0, 1000.0, 5000.0, 20000.0):
                for r2 in (None, 0, 1, 8, 9, 10, 14, 15, 31):
                    grid.append(dict(sr=sr, lf=lf, hf=hf, r2=r2))
    rng = np.random.default_rng(0)
    return [grid[i] for i in rng.choice(len(grid), 300, replace=False)]


@pytest.mark.parametrize("kind", PO.KINDS)
def test_statuses_match_reference(product_lib, ref_lib, kind):
    """new accepts exactly what the oracle accepts, refuses the rest with the oracle's status, and calTimeLength agrees
    with the reference wherever both build the object"""
    seen = set()
    for kw in _grid():
        for slide in (None, 700):
            p = PO.params(kind, **kw, slide=slide)
            st_p, o_p = PC.c_new(product_lib, kind, **kw, slide=slide)
            assert st_p == p["status"], (kw, slide, st_p, p["status"])
            seen.add(st_p)
            if st_p:
                assert not o_p
                continue
            st_r, o_r = PC.c_new(ref_lib, kind, **kw, slide=slide)
            assert st_r == 0
            for n in (0, 1, p["n"] - 1, p["n"], p["n"] + 1, p["n"] + p["slide"], 5 * p["n"] + 3, 100000):
                got = PC.c_time_length(product_lib, kind, o_p, n)
                assert got == PC.time_length(n, p["n"], p["slide"]) == PC.c_time_length(ref_lib, kind, o_r, n)
            PC.c_free(product_lib, kind, o_p)
            PC.c_free(ref_lib, kind, o_r)
    assert seen == {0, -2, -3}, seen


@pytest.mark.parametrize("kind", PO.KINDS)
def test_streaming_in_the_reference(kind):
    """isContinue: pieces of a clip (some shorter than a frame) give the frames of one call over the clip, with a slide
    below n and one above it (a negative carry)"""
    lib = ref_lib_or_none()
    if lib is None:
        pytest.skip("needs the reference build")
    x = PC.signal("glide", 40000, 16000, 5)
    for r2, slide in ((11, 512), (10, 1500)):
        st, whole = PC.c_new(lib, kind, sr=16000, r2=r2, slide=slide)
        want = PC.c_pitch(lib, kind, whole, x)
        st, o = PC.c_new(lib, kind, sr=16000, r2=r2, slide=slide, cont=1)
        got = PC.c_stream(lib, kind, o, x, (700, 3000, 100, 9000, 1, 27199))
        assert np.array_equal(got, want), (r2, slide)
        PC.c_free(lib, kind, o)
        PC.c_free(lib, kind, whole)


def test_cep_window_rule():
    """CEP keeps Hamm for any window after it: Blackman gives the Hamm outputs in the reference"""
    lib = ref_lib_or_none()
    if lib is None:
        pytest.skip("needs the reference build")
    x = PC.signal("tones", 20000, 32000, 3)
    outs = []
    for wt in (PO.W_HAMM, PO.W_BLACKMAN, PO.W_HANN):
        st, o = PC.c_new(lib, "cep", r2=12, slide=1024, wt=wt)
        outs.append(PC.c_pitch(lib, "cep", o, x))
        PC.c_free(lib, "cep", o)
    assert np.array_equal(outs[0], outs[1]) and not np.array_equal(outs[0], outs[2])
    assert PO.params("cep", wt=PO.W_BLACKMAN)["wt"] == PO.W_HAMM


def test_refusals(product_lib):
    """radix2Exp above 14, the reference's overruns (NCF maxIndex >= n, CEP maxIndex > 2n - 1), NCF minIndex < 1 and an
    empty lag range are refused at construction with a status and a reason; the object pointer stays NULL"""
    L = product_lib
    for kind, kw, st, what in (("ncf", dict(r2=15), -2, b"largest supported is 14"),
                               ("cep", dict(r2=30), -2, b"largest supported is 14"),
                               ("ncf", dict(r2=9), -3, b"is not below n"),
                               ("ncf", dict(sr=44100, r2=10), -3, b"is not below n"),
                               ("cep", dict(r2=8), -3, b"past the 2n"),
                               ("ncf", dict(sr=900, lf=100.0), -3, b"negative count"),
                               ("ncf", dict(lf=3000.0), -3, b"is empty"),
                               ("cep", dict(lf=3000.0), -3, b"is empty")):
        p = PO.params(kind, **kw)
        assert p["status"] == st, (kind, kw, p["status"])
        s, o = PC.c_new(L, kind, **kw)
        assert s == st and not o, (kind, kw, s)
        assert what in L.afb200_lastError(), L.afb200_lastError()
    for kind, r2 in (("ncf", 10), ("cep", 9)):                          # just inside the bounds: 1000 < 1024
        s, o = PC.c_new(L, kind, r2=r2)
        assert s == 0
        PC.c_free(L, kind, o)
    s, o = PC.c_new(L, "cep", r2=1, sr=8000, lf=3000.0, hf=3500.0)       # n = 2: the default slide n/4 = 0 becomes 1
    assert s == 0 and PC.c_time_length(L, "cep", o, 10) == 9
    PC.c_free(L, "cep", o)
    for kind in PO.KINDS:
        s, o = PC.c_new(L, kind, r2=12)
        assert (PC.c_pitch(L, kind, o, np.ones(4095, np.float32), fill=7.0, extra=4) == 7).all()
        v = np.zeros(4, np.float32)
        batch = getattr(L, PC.prefix(kind) + "_pitchBatch")
        assert batch(o, None, 8192, 1, v.ctypes.data, 0, None) != 0
        assert b"bad argument" in L.afb200_lastError()
        assert batch(o, v.ctypes.data, 4, -1, v.ctypes.data, 0, None) != 0
        PC.c_free(L, kind, o)
        PC.c_free(L, kind, None)
        getattr(L, PC.prefix(kind) + "_pitch")(None, None, 0, None)
        assert PC.c_time_length(L, kind, None, 100000) == 0


@pytest.mark.parametrize("kind", PO.KINDS)
def test_pitch_symbols_exported_and_bound(product_lib, kind):
    from audioflux_b200 import capi
    pre = PC.prefix(kind)
    check_symbols(product_lib, f"afb200_pitch_{kind}.h", pre + "_",
                  capi.PITCH_NCF_API if kind == "ncf" else capi.PITCH_CEP_API,
                  {pre + s for s in ("_new", "_calTimeLength", "_pitch", "_enableDebug", "_free")}, {pre + "_pitchBatch"})


def test_python_classes(product_lib):
    import audioflux_b200 as af
    for cls, win in ((af.PitchNCF, af.WindowType.RECT), (af.PitchCEP, af.WindowType.HAMM)):
        h = cls()
        assert (h.samplate, h.low_fre, h.high_fre, h.radix2_exp, h.slide_length, h.window_type, h.fft_length) == \
            (32000, 32.0, 2000.0, 12, 1024, win, 4096)
        assert h.cal_time_length(160000) == (160000 - 4096) // 1024 + 1 and h.cal_time_length(4095) == 0
        with pytest.raises(ValueError, match="status -2"):
            cls(radix2_exp=15)
        with pytest.raises(ValueError, match="at least one dimension"):
            h.pitch(np.float32(1))
        assert h.pitch(np.zeros((2, 3, 100), np.float32)).shape == (2, 3, 0)
        assert h.pitch_batch(np.zeros((0, 8000), np.float32)).shape == (0, 4)
        from audioflux_b200.lib import AfB200Error
        if product_lib.afb200_deviceCount() <= 0:          # no CPU fallback: the compute call fails loudly
            with pytest.raises(AfB200Error, match="no CUDA device"):
                h.pitch(np.ones(8000, np.float32))
    with pytest.raises(ValueError, match="low_fre"):
        af.PitchCEP(low_fre=300.0, high_fre=200.0)
    af.PitchNCF(low_fre=300.0, high_fre=200.0)             # the reference's class takes it: both ends fall back
    with pytest.raises(ValueError, match="status -3: .*is not below n"):
        af.PitchNCF(radix2_exp=9)
    with pytest.raises(ValueError, match="status -3: .*past the 2n"):
        af.PitchCEP(radix2_exp=8)
    with pytest.raises(ValueError, match="status -3: .*negative count"):
        af.PitchNCF(samplate=900)


if __name__ == "__main__":
    import sys
    if ref_lib_or_none() is None:
        sys.exit("oracle/_ref/libaudioflux_ref.so not built")
    print(f"{GOLD.name}: {GOLD.write()} arrays")
