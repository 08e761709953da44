"""CPU tier: the extended-precision references of tests/accuracy.py are what they claim to be."""
import numpy as np
import pytest

from accuracy import X_SHIFT, biquad_err, biquad_truth, dyadic_signal, dyadic_taps, exact_conv, nerr


def _int_conv(kx, kh):
    return np.array([np.convolve(kx[:, c], kh[:, c if kh.shape[1] > 1 else 0]) for c in range(kx.shape[1])]).T


@pytest.mark.parametrize("taps,frames,shared", [(1, 50, True), (37, 200, False), (500, 300, False), (1000, 4000, True)])
def test_exact_conv_equals_integer_convolution(taps, frames, shared):
    rng = np.random.default_rng(taps)
    C, S = 3, 15
    x = dyadic_signal(rng, frames, C)
    h = dyadic_taps(rng.standard_normal((taps, 1 if shared else C)), S)
    kx = (x * 2.0 ** X_SHIFT).astype(np.int64)
    kh = (h * 2.0 ** S).astype(np.int64)
    want = _int_conv(kx, kh)[:frames] * 2.0 ** -(X_SHIFT + S)
    got = exact_conv(x, h[:, 0] if shared else h, S)
    assert np.array_equal(got, want)


def test_exact_conv_selector_and_latency():
    rng = np.random.default_rng(1)
    C, S, taps, frames, lat = 5, 12, 300, 1000, 123
    sel = [1, 0, 1, 1, 0]
    x = dyadic_signal(rng, frames, C)
    h = dyadic_taps(rng.standard_normal((taps, sum(sel))), S)
    got = exact_conv(x, h, S, selector=sel, latency=lat)
    kx = (x * 2.0 ** X_SHIFT).astype(np.int64)
    kh = (h * 2.0 ** S).astype(np.int64)
    k = 0
    for c in range(C):
        if not sel[c]:
            assert np.array_equal(got[:, c], x[:, c])
            continue
        full = np.convolve(kx[:, c], kh[:, k]) * 2.0 ** -(X_SHIFT + S)
        k += 1
        assert np.array_equal(got[:lat, c], np.zeros(lat))
        assert np.array_equal(got[lat:, c], full[:frames - lat])


def test_exact_conv_full_size_budget_holds():
    """131072 taps of full-scale numerators against 2^18 frames of full-scale input: still on the grid."""
    rng = np.random.default_rng(2)
    x = dyadic_signal(rng, 1 << 18, 1)
    h = dyadic_taps(rng.uniform(-1, 1, 131072), 12)
    y = exact_conv(x, h, 12)
    assert y.shape == x.shape


def test_exact_conv_trips_when_the_bit_budget_is_exceeded():
    rng = np.random.default_rng(3)
    x = dyadic_signal(rng, 1000, 1)
    with pytest.raises(AssertionError, match="grid"):
        exact_conv(x + 2.0 ** -20, np.ones(4), 0)
    # on the grid, but numerators of 2^40 on 4096 taps: outputs need far more than 53 bits
    h = rng.integers(-2 ** 40, 2 ** 40, 4096).astype(np.float64)
    with pytest.raises(AssertionError, match="off the grid"):
        exact_conv(dyadic_signal(rng, 20000, 1), h, 0)


def _coefs():
    from oracle import restate  # noqa: F401  (the oracle package must import on the CPU tier)
    # RBJ lowpasses, 10 Hz at 192 kHz (Q 0.707) and 1 kHz at 48 kHz (Q 1.4) (c0..c4, a0-normalised)
    out = []
    for f0, fs, q in ((10.0, 192000.0, 0.707), (1000.0, 48000.0, 1.4)):
        w0 = 2 * np.pi * f0 / fs
        cs, sn = np.cos(w0), np.sin(w0)
        al = sn / (2 * q)
        a0 = 1 + al
        out.append([(1 - cs) / 2 / a0, (1 - cs) / a0, (1 - cs) / 2 / a0, -2 * cs / a0, (1 - al) / a0])
    return np.array(out)


def test_fp64_lfilter_agrees_with_the_restated_recurrence():
    from scipy.signal import lfilter
    from oracle import restate
    rng = np.random.default_rng(4)
    x = rng.standard_normal((3000, 2)) * 0.3
    coefs = _coefs()
    want = restate.biquad_cascade(x, coefs)
    got = x.copy()
    for k in coefs:
        got = lfilter(k[:3], [1.0, k[3], k[4]], got, axis=0)
    assert nerr(got, want)[0] <= 1e-13


def test_long_double_truth_is_closer_to_50_digit_arithmetic():
    """On a short input, the long-double cascade is at least as close to a 50-digit run as the FP64 recurrence."""
    import mpmath
    from oracle import restate
    rng = np.random.default_rng(5)
    x = np.concatenate([np.full(300, 0.9), rng.standard_normal(300) * 0.3])[:, None]
    coefs = _coefs()
    mpmath.mp.dps = 50
    y = [mpmath.mpf(float(v)) for v in x[:, 0]]
    for k in coefs:
        c = [mpmath.mpf(float(v)) for v in k]
        m0 = m1 = mpmath.mpf(0)
        for i, s in enumerate(y):
            r = c[0] * s + m0
            m0 = m1 + c[1] * s - c[3] * r
            m1 = c[2] * s - c[4] * r
            y[i] = r
    exact = np.array([mpmath.mpf(v) for v in y], dtype=object)
    ld = biquad_truth(x, coefs)[:, 0]
    f64 = restate.biquad_cascade(x, coefs)[:, 0]
    e_ld = max(abs(mpmath.mpf(float(a)) + mpmath.mpf(float(a - np.longdouble(float(a)))) - b) for a, b in zip(ld, exact))
    e_64 = max(abs(mpmath.mpf(float(a)) - b) for a, b in zip(f64, exact))
    assert e_ld <= e_64
    assert e_ld < 1e-15 * float(np.max(np.abs(f64)))
    assert biquad_err(f64, ld) > 0.0
