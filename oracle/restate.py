"""oracle/restate.py -- TEST INFRASTRUCTURE ONLY (never imported by the product).

numpy restatement of the reference's hot-path arithmetic, one function per reference routine,
each citing the file:line it follows (paths under /root/reference).  It is validated against
the compiled reference (oracle/_ref, see oracle/ref.py) by tests/test_oracle.py and against the
committed golden vectors under tests/golden/, and is the fallback checker when the compiled
reference is not available.

Parity status: the reference ships no tests or golden vectors for this path (SURVEY.md 4, 8c),
so the pin is the reference's own code compiled here (oracle/Makefile) -- and its FFT backend is
oracle/fftw3_shim.c, not FFTW3 (un-vendored, version unpinned, absent).
"""
import math

import numpy as np


# --------------------------------------------------------------------------------------------
# sgen.c:44-69,158-167 -- the mandated input: sine or exponential sweep, same value on every channel
# --------------------------------------------------------------------------------------------
def sgen_sine(fs, channels, frames, freq0=440.0, freq1=None, offset=0):
    pos = np.arange(offset, offset + frames, dtype=np.float64)
    t = pos / fs
    w0 = 2.0 * math.pi * freq0
    if freq1 is None or freq1 == freq0:
        s = np.sin(w0 * t)
    else:
        v = math.log(freq1 / freq0) / (frames / fs)   # sgen.c:162-164 (sweep over the generator length)
        s = np.sin(w0 / v * (np.exp(t * v) - 1.0))
    return np.repeat(s[:, None], channels, axis=1)


# --------------------------------------------------------------------------------------------
# biquad.h:76-92 (TDF-II) applied per stage in place, biquad.c:296-315
# --------------------------------------------------------------------------------------------
def biquad_cascade(x, coefs, state=None):
    """x [frames, C]; coefs [S, C, 5] = c0..c4; state [S, C, 2] (m0, m1), updated in place."""
    x = np.array(x, dtype=np.float64, copy=True)
    coefs = np.asarray(coefs, dtype=np.float64)
    S, C = coefs.shape[0], x.shape[1]
    if coefs.ndim == 2:
        coefs = np.repeat(coefs[:, None, :], C, axis=1)
    if state is None:
        state = np.zeros((S, C, 2))
    for st in range(S):
        c0, c1, c2, c3, c4 = (coefs[st, :, k] for k in range(5))
        m0, m1 = state[st, :, 0].copy(), state[st, :, 1].copy()
        for i in range(x.shape[0]):
            s = x[i]
            r = c0 * s + m0
            m0 = m1 + c1 * s - c3 * r
            m1 = c2 * s - c4 * r
            x[i] = r
        state[st, :, 0], state[st, :, 1] = m0, m1
    return x


# --------------------------------------------------------------------------------------------
# fir.c:43-62 / fir.c:109-149 / fir_p.c:64-181: all three compute the linear convolution
# (fir's FFT path additionally delays by len = next_fast_fftw_len(taps), fir.c:298, util.c:434-458)
# --------------------------------------------------------------------------------------------
def next_fast_fftw_len(n):
    """util.c:434-458: smallest 2^a 3^b 5^c 7^d >= n."""
    while True:
        m = n
        for p in (2, 3, 5, 7):
            while m % p == 0:
                m //= p
        if m == 1:
            return n
        n += 1


def fir_stream(x, taps, selector=None, latency=0, out_frames=None):
    """x [frames, C]; taps [T] or [T, fc] (column k -> k-th selected channel, fir.c:348-356).
    Returns the first `out_frames` (default frames) frames of the stream the effect emits."""
    x = np.asarray(x, dtype=np.float64)
    taps = np.asarray(taps, dtype=np.float64)
    if taps.ndim == 1:
        taps = taps[:, None]
    frames, C = x.shape
    n_out = frames if out_frames is None else out_frames
    y = np.zeros((n_out, C))
    k = 0
    nfft = 1
    while nfft < frames + taps.shape[0]:
        nfft *= 2
    for c in range(C):
        if selector is not None and not selector[c]:
            y[:min(n_out, frames), c] = x[:n_out, c]
            continue
        h = taps[:, 0] if taps.shape[1] == 1 else taps[:, k]
        k += 1
        full = np.fft.irfft(np.fft.rfft(x[:, c], nfft) * np.fft.rfft(h, nfft), nfft)[:frames + taps.shape[0] - 1]
        seg = np.concatenate([np.zeros(latency), full])
        m = min(n_out, seg.shape[0])
        y[:m, c] = seg[:m]
    return y


# hilbert.c:65-77
def hilbert_taps(taps, angle=-math.pi / 2):
    h = np.zeros(taps)
    w_h, w_d = math.sin(-angle), math.cos(-angle)
    for i in range(taps):
        k = i - taps // 2
        if k == 0:
            h[i] = w_d
        elif k % 2 == 0:
            h[i] = 0.0
        else:
            xx = 2.0 * math.pi * i / (taps - 1)
            h[i] = w_h * 2.0 / (math.pi * k) * (0.42 - 0.5 * math.cos(xx) + 0.08 * math.cos(2.0 * xx))
    return h


# --------------------------------------------------------------------------------------------
# resample.c
# --------------------------------------------------------------------------------------------
_ALBRECHT9 = [2.318028013590306028393e-1, 3.932575471789488615081e-1, 2.385434764970747429454e-1,
              1.014370437785239811268e-1, 2.911516061918003918645e-2, 5.280988177252078698806e-3,
              5.382909093381945363528e-4, 2.442086527507867730168e-5, 2.706153764205043532817e-7]
_M_FACT = 17.7822


def _window(x):
    """resample.c:52-80"""
    if x >= 1.0 or x <= 0.0:
        return 0.0
    w = _ALBRECHT9[0]
    for i in range(1, 9):
        c = -_ALBRECHT9[i] if (i & 1) else _ALBRECHT9[i]
        w += c * math.cos(2 * i * math.pi * x)
    return w


def _ratio_mult_ceil(v, n, d):
    """util.h:180-184"""
    r = v * n
    return r // d + (1 if r % d else 0)


class Resampler:
    """resample.c:213-386 (init), :89-152 (run), :154-161 (reset), :163-188 (drain2)."""

    def __init__(self, fs_in, fs_out, channels, bw=0.939):
        mx, mn = max(fs_in, fs_out), min(fs_in, fs_out)
        g = math.gcd(fs_in, fs_out)
        self.n, self.d = fs_out // g, fs_in // g
        maxf, minf = max(self.n, self.d), min(self.n, self.d)
        m = int(math.floor(2.0 * _M_FACT * mx / (mn * (1.0 - bw)) + 0.5))          # :281
        width = _M_FACT * mx / m
        fc = (mn - width) / mx
        sinc_os = min(minf, 2)
        fc_os = fc / sinc_os
        m_os = (m + 1) * sinc_os - 1
        len_mult = (m + 1) // maxf + (1 if (m + 1) % maxf else 0)                    # :294-295
        if len_mult > 16:
            fast = next_fast_fftw_len(len_mult)
            if fast != len_mult and (self.n <= 16 or self.d <= 16 or next_fast_fftw_len(self.n) == self.n
                                     or next_fast_fftw_len(self.d) == self.d):
                len_mult = fast
        sinc_len = maxf * len_mult * sinc_os
        self.in_len, self.out_len = self.d * len_mult, self.n * len_mult
        self.tmp_fr_len = maxf * len_mult + 1
        self.sinc_fr_len = sinc_len + 1
        if fs_out == mx:
            self.out_delay = m // 2
        else:
            self.out_delay = int(math.floor((m // 2) * (self.n / self.d) + 0.5))       # :316
        sinc = np.zeros(sinc_len * 2)
        for i in range(1, m_os):                                                      # :363-364
            xx = (i * 2 - m_os) / 2.0
            s = fc_os if abs(xx) < 1e-9 else math.sin(math.pi * fc_os * xx) / (math.pi * xx)
            sinc[i] = s * _window(i / m_os)
        self.sinc = sinc                    # kept for the extended-precision tap table (tests/accuracy.py)
        self.sinc_fr = np.fft.rfft(sinc)
        self.m = m
        self.C = channels
        self.input = np.zeros((channels, self.in_len * 2))
        self.output = np.zeros((channels, self.out_len * 2))
        self.overlap = np.zeros((channels, self.out_len))
        self.in_buf_pos = self.out_buf_pos = 0
        self.has_output = 0
        self.is_draining = 0
        self.drain_pos = self.drain_frames = 0

    def _block(self):
        """resample.c:110-142 for every channel."""
        for c in range(self.C):
            X = np.fft.rfft(self.input[c])
            Y = np.zeros(self.tmp_fr_len, dtype=np.complex128)
            Y[0] = X[0] * self.sinc_fr[0]
            k, j, l, d1, d2 = 1, 1, 1, 1, 1
            while True:
                s = X[j] if d1 == 1 else np.conj(X[j])
                Y[l] += s * self.sinc_fr[k] if d2 == 1 else np.conj(s * self.sinc_fr[k])
                if k + 1 == self.sinc_fr_len:
                    break
                if l == self.out_len:
                    Y[l] += s * self.sinc_fr[k]
                elif l == 0:
                    Y[l] += np.conj(s * self.sinc_fr[k])
                j += d1
                l += d2
                if j == 0:
                    d1 = 1
                elif j == self.in_len:
                    d1 = -1
                if l == 0:
                    d2 = 1
                elif l == self.out_len:
                    d2 = -1
                k += 1
            # c2r of 2*out_len points, unnormalised (irfft divides by its length), then / (2 in_len)
            o = np.fft.irfft(Y[:self.out_len + 1], self.out_len * 2) * (self.out_len * 2) / (self.in_len * 2)
            o[:self.out_len] += self.overlap[c]
            self.overlap[c] = o[self.out_len:]
            self.output[c] = o

    def run(self, x):
        x = np.asarray(x, dtype=np.float64)
        frames = x.shape[0]
        max_o = _ratio_mult_ceil(frames, self.n, self.d)
        out = np.zeros((max_o, self.C))
        i = o = 0
        while i < frames:
            while self.in_buf_pos < self.in_len and i < frames:
                self.input[:, self.in_buf_pos] = x[i]
                i += 1
                self.in_buf_pos += 1
            while self.out_buf_pos < self.out_len and o < max_o and self.has_output:
                out[o] = self.output[:, self.out_buf_pos]
                o += 1
                self.out_buf_pos += 1
            if self.in_buf_pos == self.in_len and (not self.has_output or self.out_buf_pos == self.out_len):
                self._block()
                self.in_buf_pos = self.out_buf_pos = 0
                if not self.has_output:
                    self.out_buf_pos = self.out_delay
                    self.has_output = 1
        return out[:o]

    def reset(self):
        """resample.c:154-161: the drain counters are left alone."""
        self.in_buf_pos = self.out_buf_pos = 0
        self.has_output = 0
        self.overlap[:] = 0.0

    def drain2(self, frames):
        if not self.has_output and self.in_buf_pos == 0:
            return None
        if not self.is_draining:
            if self.has_output:
                self.drain_frames += self.out_delay
                self.drain_frames += self.out_len - self.out_buf_pos
            self.drain_frames += _ratio_mult_ceil(self.in_buf_pos, self.n, self.d)
            self.is_draining = 1
        if self.drain_pos < self.drain_frames:
            y = self.run(np.zeros((frames, self.C)))
            self.drain_pos += y.shape[0]
            if self.drain_pos > self.drain_frames:
                y = y[:y.shape[0] - (self.drain_pos - self.drain_frames)]
            return y
        return None

    def process(self, x, block):
        outs, counts = [], []
        for i in range(0, x.shape[0], block):
            y = self.run(x[i:i + block])
            outs.append(y)
            counts.append(y.shape[0])
        while True:
            y = self.drain2(block)
            if y is None:
                break
            outs.append(y)
            counts.append(y.shape[0])
        return np.concatenate(outs, axis=0), counts


# --------------------------------------------------------------------------------------------
# seeded impulse responses of the benchmark configs (SURVEY.md 8d), Park-Miller util.h:127-148
# --------------------------------------------------------------------------------------------
def pm_rand1_sequence(seed, count):
    """pm_rand1_r (util.h:127-148) is x -> 48271 x mod (2^31 - 1); the k-th output is
    seed * 48271^k mod (2^31 - 1), built here by doubling so that long sequences stay vectorised."""
    M = np.uint64(0x7fffffff)
    pw = np.array([48271], dtype=np.uint64)          # 48271^1 .. 48271^len
    while pw.shape[0] < count:
        pw = np.concatenate([pw, (pw * pw[-1]) % M])
    return ((pw[:count] * np.uint64(seed % 0x7fffffff)) % M).astype(np.int64)


def bench_ir(taps, channel=0):
    """h[n] = u_n exp(-6.9 n/taps), u_n = 2 r_n/2147483647 - 1 (pm_rand1_r, seed 1+channel),
    scaled to sum|h| = 0.5."""
    r = pm_rand1_sequence(1 + channel, taps).astype(np.float64)
    u = 2.0 * r / 2147483647.0 - 1.0
    h = u * np.exp(-6.9 * np.arange(taps) / taps)
    return h * (0.5 / np.sum(np.abs(h)))
