"""CPU tier: the extended-precision references of tests/accuracy.py are what they claim to be."""
import numpy as np
import pytest

from accuracy import (RS_RATIOS, X_SHIFT, RsPacing, biquad_err, biquad_truth, dyadic_signal, dyadic_taps, exact_conv, nerr,
                      resample_taps_truth, resample_truth, rs_counts, rs_nerr, taps_from_sinc)


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


# ------------------------------------------------------------------------------------------------------------
# Resample
# ------------------------------------------------------------------------------------------------------------
def _ld_to_mp(a):
    """A long double as an mpmath number (its two double parts)."""
    import mpmath
    hi = float(a)
    return mpmath.mpf(hi) + mpmath.mpf(float(a - np.longdouble(hi)))


def _mp_taps(sinc, n, in_len, entries, dps=40):
    """G[ph][t] at the (ph, t) in `entries` by the cosine sum of resample.cu's header, in `dps`-digit arithmetic:
    S = DFT_2K(sinc), g(tau) = 1/(2 in_len) [S_0 + 2 sum_{k<K} Re(S_k e^{i th k tau}) + Re(S_K e^{i th K tau})]."""
    import mpmath
    mpmath.mp.dps = dps
    K = len(sinc) // 2
    cs = [mpmath.cospi(mpmath.mpf(j) / K) for j in range(2 * K)]
    sn = [mpmath.sinpi(mpmath.mpf(j) / K) for j in range(2 * K)]
    nz = [(i, mpmath.mpf(float(v))) for i, v in enumerate(sinc) if v != 0.0]
    S = [(mpmath.fsum(v * cs[(i * k) % (2 * K)] for i, v in nz), -mpmath.fsum(v * sn[(i * k) % (2 * K)] for i, v in nz))
         for k in range(K + 1)]
    Pd = 2 * in_len * n
    out = []
    for ph, t in entries:
        tau = ph + t * n
        acc = mpmath.mpf(0)
        for k in range(1, K + 1):
            a = mpmath.mpf(2 * ((k * tau) % Pd)) / Pd
            term = S[k][0] * mpmath.cospi(a) - S[k][1] * mpmath.sinpi(a)
            acc += term / 2 if k == K else term
        out.append((S[0][0] + 2 * acc) / (2 * in_len))
    return out


@pytest.mark.parametrize("fs_in,fs_out", [(32000, 48000), (48000, 32000)])
def test_resample_taps_truth_matches_40_digit_cosine_sum(fs_in, fs_out):
    """The long-double tap table against the cosine sum in 40 digits at 50 seeded entries (3:2 and 2:3 at
    bandwidth 0.7, where K is small): the 1 / (2 in_len) scale and the phase / tap indexing."""
    from oracle import restate
    r = restate.Resampler(fs_in, fs_out, 1, bw=0.7)
    G = resample_taps_truth(fs_in, fs_out, 0.7)
    assert G.shape == (r.n, r.in_len)
    rng = np.random.default_rng(fs_in)
    entries = [(int(rng.integers(r.n)), int(rng.integers(r.in_len))) for _ in range(50)]
    want = _mp_taps(r.sinc, r.n, r.in_len, entries)
    peak = float(np.max(np.abs(G)))
    err = max(abs(_ld_to_mp(G[ph, t]) - w) for (ph, t), w in zip(entries, want))
    assert err <= 1e-17 * peak, err / peak


@pytest.mark.parametrize("K,n,in_len", [(12, 3, 8), (10, 1, 10), (10, 2, 5)])
def test_taps_from_sinc_weights_the_last_bin_as_the_cosine_sum(K, n, in_len):
    """A random 2K-point 'sinc' makes S_K as large as the other bins (a designed lowpass leaves it near 1e-20 of
    ||G||, too small to see): the last bin's weight, with K below the Nyquist bin Pd / 2 and (10, 1, 10; 10, 2, 5)
    equal to it, and the whole table, against 40 digits."""
    rng = np.random.default_rng(K + n)
    sinc = rng.standard_normal(2 * K)
    G = taps_from_sinc(sinc, n, in_len)
    entries = [(ph, t) for ph in range(n) for t in range(in_len)]
    want = _mp_taps(sinc, n, in_len, entries)
    err = max(abs(_ld_to_mp(G[ph, t]) - w) for (ph, t), w in zip(entries, want))
    assert err <= 1e-17 * float(np.max(np.abs(G))), err


def _ragged(rng, N, in_len):
    """Cut points of a ragged stream: 1, 7, in_len - 1, in_len, in_len + 1 frames and random sizes."""
    sizes = [1, 7, in_len - 1, in_len, in_len + 1]
    while sum(sizes) < N:
        sizes.append(int(rng.integers(1, 2 * in_len)))
    cuts = np.cumsum([0] + sizes)
    return [int(c) for c in cuts[cuts < N]] + [N]


@pytest.mark.parametrize("bw", [0.7, 0.939, 0.99])
@pytest.mark.parametrize("rates", RS_RATIOS)
def test_resample_truth_matches_the_fp64_reference(have_ref, rates, bw):
    """The LPTV sum from the long-double table, against the reference algorithm in FP64 (restate.Resampler, and the
    compiled reference where it is built) on ragged calls with the drain: ties the formula, out_delay and the drain
    to the reference's block-FFT form (outputs past 3000 sampled).  Bound: normalized RMS <= 2e-15 (the FP64 reference is ~4e-16 from the truth);
    every per-call count as rs_counts replays it."""
    from oracle import restate
    fi, fo = rates
    r = restate.Resampler(fi, fo, 2, bw=bw)
    rng = np.random.default_rng(fi + fo + int(1000 * bw))
    N = 2 * r.in_len + 300
    x = dyadic_signal(rng, N, 2)
    x[:, 1] = 0.9 * np.sin(2 * np.pi * 0.3 * min(fi, fo) * np.arange(N) / fi)
    cuts = _ragged(rng, N, r.in_len)
    block = 997
    refs = [r]
    if have_ref:
        from oracle import ref
        refs.append(ref.RefChain("resample %s %d" % (bw, fo), fi, 2))
    G = resample_taps_truth(fi, fo, bw)
    counts, drains = rs_counts(fi, fo, np.diff(cuts), block, bw)
    for rr in refs:
        outs = [rr.run(x[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
        assert [o.shape[0] for o in outs] == counts
        if rr is r:
            while (y := r.drain2(block)) is not None:
                outs.append(y)
        else:
            outs += rr.drain(block)
        assert [o.shape[0] for o in outs[len(counts):]] == drains
        got = np.concatenate(outs)
        # every output of short streams; of long ones (large n or bandwidth) the first and last 200 and a seeded sample
        rows = np.arange(got.shape[0])
        if rows.size > 3000:
            rows = np.unique(np.concatenate([rows[:200], rows[-200:], rng.choice(rows, 2600, replace=False)]))
        want = resample_truth(x, fi, fo, bw, got.shape[0], rows=rows, G=G)
        e = rs_nerr(got[rows], want, x, G)
        assert e[0] <= 2e-15, (rr, e)


@pytest.mark.parametrize("rates,bw", [((44100, 48000), 0.939), ((48000, 8000), 0.7), ((8000, 44100), 0.99)])
def test_rs_pacing_matches_the_reference_counts(rates, bw):
    """Per-call counts of RsPacing against restate.Resampler: 1-frame calls, tiny calls then a large one, a drain,
    reset() mid-stream (the drain counters persist, so a second drain after a reset is dry), and a drain after a
    reset before the first block."""
    from oracle import restate
    fi, fo = rates
    r = restate.Resampler(fi, fo, 1, bw=bw)
    p = RsPacing(fi, fo, bw)
    L = r.in_len
    script = ([("run", 1)] * 40 + [("run", 5)] * 200 + [("run", 3 * L + 17)] + [("reset", 0), ("run", L - 1), ("drain", 7)]
              + [("drain", 1), ("drain", 4096)] * 3 + [("reset", 0), ("run", 1), ("run", 8192)] + [("drain", 1000)] * 3
              + [("reset", 0), ("drain", 5)])
    for op, f in script:
        if op == "run":
            assert p.run(f) == r.run(np.zeros((f, 1))).shape[0]
        elif op == "reset":
            p.reset()
            r.reset()
        else:
            y = r.drain2(f)
            assert p.drain(f) == (None if y is None else y.shape[0])
    assert p.is_draining and p.drain_frames > 0
