"""Extended-precision references and one error metric for the accuracy tests (test code only; the product never
imports it).

FIR: `exact_conv` is the exact linear convolution of dyadic signals.  x = k 2^-12 with |k| <= 2^11 and
h = j 2^-S with |j| <= 2^12, so every output sample is an integer multiple of 2^-(12+S) whose numerator needs
about 23 + log2(taps) bits: at 131072 taps and beyond it is still far inside the 53 bits of a double.  The
FP64 FFT convolution of the integer numerators is then within a small fraction of a unit of the exact
integers, and rounding to the grid recovers them exactly.

Biquad: `biquad_truth` runs the same double coefficients through scipy's lfilter in 80-bit long double.

Errors are reported as nerr = rms(got - want) / scale (and nmax with the max): for FIR, scale = rms(x) ||h||_2
per channel, elsewhere scale = rms(want).
"""
import os
from contextlib import contextmanager

import numpy as np

X_SHIFT = 12       # x = k 2^-12
X_MAX = 1 << 11    # |k| <= 2^11
H_MAX = 1 << 12    # |j| <= 2^12
U = 2.0 ** -53     # unit roundoff of FP64


def dyadic_signal(rng, frames, channels, amp=0.5):
    """Uniform white noise of peak `amp` (<= 0.5) on the grid k 2^-12."""
    kmax = min(int(amp * (1 << X_SHIFT)), X_MAX)
    return rng.integers(-kmax, kmax + 1, size=(frames, channels)).astype(np.float64) * 2.0 ** -X_SHIFT


def dyadic_taps(h, shift):
    """Round `h` (any shape; its peak is scaled to 1) to the grid j 2^-shift, |j| <= 2^12."""
    h = np.asarray(h, dtype=np.float64)
    peak = np.max(np.abs(h))
    return np.round(h / peak * H_MAX) * 2.0 ** -shift


def _numerators(a, shift, what):
    k = np.asarray(a, dtype=np.float64) * 2.0 ** shift
    assert np.array_equal(k, np.round(k)), "%s is not on the 2^-%d grid" % (what, shift)
    return k


def exact_conv(x, h, h_shift, selector=None, latency=0):
    """Exact linear convolution of dyadic x [frames, C] with dyadic taps h [T] or [T, fc] (column k -> k-th
    selected channel), delayed by `latency` frames, first `frames` frames: the stream restate.fir_stream describes.
    Unselected channels pass through.  Fails when the FP64 FFT lands more than 0.05 units off the output grid,
    i.e. when the operands exceed the bit budget."""
    x = np.asarray(x, dtype=np.float64)
    frames, C = x.shape
    h = np.asarray(h, dtype=np.float64)
    if h.ndim == 1:
        h = h[:, None]
    kx = _numerators(x, X_SHIFT, "x")
    kh = _numerators(h, h_shift, "h")
    T = h.shape[0]
    nfft = 1
    while nfft < frames + T:
        nfft *= 2
    y = np.zeros((frames, C))
    sel = [True] * C if selector is None else [bool(s) for s in selector]
    cols = [c for c in range(C) if sel[c]]
    for c in range(C):
        if not sel[c]:
            y[:, c] = x[:, c]
    Hf = np.fft.rfft(kh, nfft, axis=0)
    n_keep = max(frames - latency, 0)
    for k, c in enumerate(cols):
        full = np.fft.irfft(np.fft.rfft(kx[:, c], nfft) * Hf[:, 0 if h.shape[1] == 1 else k], nfft)[:n_keep]
        r = np.round(full)
        dev = np.max(np.abs(full - r), initial=0.0)
        assert dev <= 0.05, "FFT result %.3g units off the grid: operands exceed the bit budget" % dev
        y[latency:, c] = r * 2.0 ** -(X_SHIFT + h_shift)
        if latency:
            y[:latency, c] = 0.0
    return y


def fir_scale(x, h, selector=None):
    """Per selected channel: rms(x_c) ||h_c||_2 (list, one entry per selected channel)."""
    x = np.asarray(x, dtype=np.float64)
    h = np.asarray(h, dtype=np.float64)
    if h.ndim == 1:
        h = h[:, None]
    cols = [c for c in range(x.shape[1]) if selector is None or selector[c]]
    return np.array([np.sqrt(np.mean(x[:, c] ** 2)) * np.linalg.norm(h[:, 0 if h.shape[1] == 1 else k])
                     for k, c in enumerate(cols)]), cols


def fir_nerr(got, want, x, h, selector=None):
    """(worst normalized RMS, worst normalized max) over the selected channels."""
    scale, cols = fir_scale(x, h, selector)
    d = np.asarray(got, dtype=np.float64)[:, cols] - np.asarray(want, dtype=np.float64)[:, cols]
    return float(np.max(np.sqrt(np.mean(d * d, axis=0)) / scale)), float(np.max(np.max(np.abs(d), axis=0) / scale))


def nerr(got, want, scale=None):
    """(rms(got - want) / scale, max|got - want| / scale); scale defaults to rms(want)."""
    d = np.asarray(got, dtype=np.float64) - np.asarray(want, dtype=np.float64)
    w = np.asarray(want, dtype=np.float64)
    if scale is None:
        scale = float(np.sqrt(np.mean(w * w)))
    return float(np.sqrt(np.mean(d * d))) / scale, float(np.max(np.abs(d), initial=0.0)) / scale


def biquad_truth(x, coefs):
    """x [frames, C]; coefs [S, 5] or [S, C, 5] (double).  The cascade in 80-bit long double: per stage,
    lfilter(b = c0..c2, a = [1, c3, c4]).  Returns long double."""
    from scipy.signal import lfilter
    y = np.asarray(x, dtype=np.float64).astype(np.longdouble)
    coefs = np.asarray(coefs, dtype=np.float64)
    if coefs.ndim == 2:
        coefs = np.repeat(coefs[:, None, :], y.shape[1], axis=1)
    for st in range(coefs.shape[0]):
        for c in range(y.shape[1]):
            k = coefs[st, c].astype(np.longdouble)
            y[:, c] = lfilter(k[:3], np.array([1.0, k[3], k[4]], dtype=np.longdouble), y[:, c])
    return y


def biquad_err(got, truth):
    """rms(got - truth) in long double, as a float."""
    d = np.asarray(got, dtype=np.float64).astype(np.longdouble) - truth
    return float(np.sqrt(np.mean(d * d)))


def biquad_within_ref(got, x, coefs):
    """Per channel: err_gpu <= max(4 err_ref64, 64 u rms(truth)), both errors against biquad_truth, err_ref64 that of
    the reference's own FP64 recurrence (restate.biquad_cascade).  Returns per channel (err_gpu, err_ref64, ratio to
    the bound), errors relative to rms(truth); asserts the bound."""
    from oracle import restate
    truth = biquad_truth(x, coefs)
    ref64 = restate.biquad_cascade(x, coefs)
    out = []
    for c in range(x.shape[1]):
        t = truth[:, c]
        e_gpu, e_ref = biquad_err(got[:, c], t), biquad_err(ref64[:, c], t)
        scale = float(np.sqrt(np.mean(t * t)))
        bound = max(4 * e_ref, 64 * U * scale)
        out.append((e_gpu / scale, e_ref / scale, e_gpu / bound))
        assert e_gpu <= bound, (c, e_gpu / scale, e_ref / scale)
    return out


@contextmanager
def env(**kw):
    """Set (or, with None, unset) environment variables for the duration of the block; the library reads its plan-time
    switches with getenv() when an operator is planned."""
    old = {k: os.environ.get(k) for k in kw}
    for k, v in kw.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
