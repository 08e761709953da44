"""Extended-precision references and one error metric for the accuracy tests (test code only; the product never
imports it).

FIR: `exact_conv` is the exact linear convolution of dyadic signals.  x = k 2^-12 with |k| <= 2^11 and
h = j 2^-S with |j| <= 2^12, so every output sample is an integer multiple of 2^-(12+S) whose numerator needs
about 23 + log2(taps) bits: at 131072 taps and beyond it is still far inside the 53 bits of a double.  The
FP64 FFT convolution of the integer numerators is then within a small fraction of a unit of the exact
integers, and rounding to the grid recovers them exactly.

Biquad: `biquad_truth` runs the same double coefficients through scipy's lfilter in 80-bit long double.

Resample: `resample_taps_truth` is the tap table G of the polyphase form (resample.cu header) in long double, built
from the reference's own sinc samples; `resample_truth` evaluates the emitted stream from it in long double, and
`RsPacing` / `rs_counts` replay the per-call frame counts in integers.

Errors are reported as nerr = rms(got - want) / scale (and nmax with the max): for FIR, scale = rms(x) ||h||_2
per channel, for resample rms(x) ||G|| per channel (`rs_nerr`), elsewhere scale = rms(want).
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


# the ratios of test_gpu_parity.test_resample_ratios: large n (640/147), sinc_os = 1 (2:1, 1:2), 1:6 and 6:1
RS_RATIOS = [(44100, 48000), (48000, 44100), (48000, 96000), (96000, 48000), (44100, 32000), (44100, 96000),
             (44100, 192000), (192000, 44100), (96000, 44100), (88200, 44100), (44100, 88200), (48000, 8000),
             (8000, 48000), (11025, 48000), (8000, 44100)]


def resample_taps_truth(fs_in, fs_out, bw=0.939):
    """The resampler's tap table G [n, in_len] in long double: G[ph][t] = g(ph + t n) with
        g(tau) = 1/(2 in_len) [S_0 + 2 sum_{k=1}^{K-1} Re(S_k e^{i th k tau}) + Re(S_K e^{i th K tau})],
    th = 2 pi / Pd, Pd = 2 in_len n, K = sinc_len, S = DFT_{2K} of the reference's windowed sinc (resample.cu header).
    That sum is a real inverse DFT of length Pd whose bins 0..K-1 hold S_k and bin K holds S_K / 2 -- or S_K itself
    when K is the Nyquist bin Pd / 2 (ratios 1:m and m:1), which the inverse transform does not double."""
    from oracle import restate
    r = restate.Resampler(fs_in, fs_out, 1, bw=bw)
    return taps_from_sinc(r.sinc, r.n, r.in_len)


def taps_from_sinc(sinc, n, in_len):
    """resample_taps_truth for any 2K-point real array `sinc` (K = len(sinc) / 2)."""
    K = len(sinc) // 2
    S = np.fft.rfft(np.asarray(sinc, dtype=np.float64).astype(np.longdouble))
    Pd = 2 * in_len * n
    B = np.zeros(Pd // 2 + 1, dtype=np.clongdouble)
    B[:K] = S[:K]
    B[K] = S[K] if 2 * K == Pd else S[K] / 2
    g = np.fft.irfft(B, Pd) * (np.longdouble(Pd) / (2 * in_len))
    return g[np.arange(n)[:, None] + np.arange(in_len)[None, :] * n]


def taps_norm(G):
    """||G|| = sqrt(mean over phases of sum_t G[ph][t]^2): the gain of the resampler on white noise."""
    G = np.asarray(G, dtype=np.float64)
    return float(np.sqrt(np.mean(np.sum(G * G, axis=1))))


def resample_truth(x, fs_in, fs_out, bw, n_out, rows=None, G=None):
    """The emitted stream of the resampler on x [frames, C] (zero before the stream and after its end, which is what
    the drain feeds): y[q] = sum_t G[(m d) mod n][t] x[floor(m d / n) - t], m = out_delay + q, for q < n_out, or
    only for the emitted indices in `rows`.  Long double, in chunks of outputs so that memory stays bounded."""
    from oracle import restate
    r = restate.Resampler(fs_in, fs_out, 1, bw=bw)
    if G is None:
        G = resample_taps_truth(fs_in, fs_out, bw)
    x = np.asarray(x, dtype=np.float64)
    N, C = x.shape
    q = np.arange(n_out) if rows is None else np.asarray(rows, dtype=np.int64)
    m = r.out_delay + q
    ph, ih = (m * r.d) % r.n, (m * r.d) // r.n
    # x with in_len zero rows in front and zeros past the end: input row i lives at i + in_len
    hi = int(ih.max(initial=0)) + 1
    xp = np.zeros((r.in_len + max(hi, N), C), dtype=np.longdouble)
    xp[r.in_len:r.in_len + N] = x
    t = np.arange(r.in_len)
    y = np.zeros((q.size, C), dtype=np.longdouble)
    step = max(1, (1 << 21) // (r.in_len * C))
    for a in range(0, q.size, step):
        idx = (ih[a:a + step] + r.in_len)[:, None] - t[None, :]
        y[a:a + step] = np.einsum("qt,qtc->qc", G[ph[a:a + step]], xp[idx])
    return y


class RsPacing:
    """The resampler's per-call frame counts in integers: resample.c:91-151 (run), :154-161 (reset, which leaves the
    drain counters alone) and :163-188 (drain2).  drain() returns None where the library reports a dry drain."""

    def __init__(self, fs_in, fs_out, bw=0.939):
        from oracle import restate
        r = restate.Resampler(fs_in, fs_out, 1, bw=bw)
        self.n, self.d, self.in_len, self.out_len, self.out_delay = r.n, r.d, r.in_len, r.out_len, r.out_delay
        self.in_buf_pos = self.out_buf_pos = self.has_output = 0
        self.is_draining = self.drain_pos = self.drain_frames = 0

    def _max_out(self, frames):
        v = frames * self.n
        return v // self.d + (1 if v % self.d else 0)

    def run(self, frames):
        mo, i, o = self._max_out(frames), 0, 0
        while i < frames:
            take = min(self.in_len - self.in_buf_pos, frames - i)
            self.in_buf_pos += take
            i += take
            if self.has_output:
                e = min(self.out_len - self.out_buf_pos, mo - o)
                self.out_buf_pos += e
                o += e
            if self.in_buf_pos == self.in_len and (not self.has_output or self.out_buf_pos == self.out_len):
                self.in_buf_pos = self.out_buf_pos = 0
                if not self.has_output:
                    self.out_buf_pos = self.out_delay
                    self.has_output = 1
        return o

    def reset(self):
        self.in_buf_pos = self.out_buf_pos = self.has_output = 0

    def drain(self, frames):
        if not self.has_output and self.in_buf_pos == 0:
            return None
        if not self.is_draining:
            if self.has_output:
                self.drain_frames += self.out_delay + self.out_len - self.out_buf_pos
            self.drain_frames += self._max_out(self.in_buf_pos)
            self.is_draining = 1
        if self.drain_pos >= self.drain_frames:
            return None
        o = self.run(frames)
        self.drain_pos += o
        return o - max(self.drain_pos - self.drain_frames, 0)


def rs_counts(fs_in, fs_out, sizes, drain_block=None, bw=0.939):
    """(per-call frame counts of calls of `sizes` frames, counts of the drain polls of `drain_block` frames that
    follow until the drain is dry; [] without a drain)."""
    p = RsPacing(fs_in, fs_out, bw)
    counts = [p.run(int(f)) for f in sizes]
    drains = []
    while drain_block:
        o = p.drain(drain_block)
        if o is None:
            break
        drains.append(o)
    return counts, drains


def rs_nerr(got, want, x, G):
    """(worst normalized RMS, worst normalized max) over channels, scale = rms(x_c) ||G|| per channel: the size of the
    output white noise of that power would have, so a stopband input whose output is tiny still gives a meaningful
    figure."""
    x = np.asarray(x, dtype=np.float64)
    scale = np.sqrt(np.mean(x * x, axis=0)) * taps_norm(G)
    d = (np.asarray(got, dtype=np.float64).astype(np.longdouble) - np.asarray(want, dtype=np.longdouble)).astype(np.float64)
    return float(np.max(np.sqrt(np.mean(d * d, axis=0)) / scale)), float(np.max(np.max(np.abs(d), axis=0) / scale))


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
