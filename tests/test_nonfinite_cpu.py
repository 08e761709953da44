"""CPU tier: the dependency windows of tests/test_gpu_nonfinite.py (accuracy.fir_nan_window, accuracy.rs_nan_windows)
against brute-force numpy models that push a NaN through the same block structure and see where it lands."""
import numpy as np
import pytest

from accuracy import fir_b0, fir_level_taps, fir_nan_window, rs_expect_launch, rs_nan_windows


def _fir_model(N, n, taps, levels):
    """Non-finite outputs of a partitioned overlap-save convolution with `levels` [{"B", "P"}] (fir_level_taps), all taps
    non-zero, input zero but for a NaN at frame n: output block m of a level sums X_{m - tap0/B - p} H_p, X_j the 2B-point
    transform of input blocks j - 1 and j."""
    x = np.zeros(N)
    x[n] = np.nan
    h = np.ones(taps)
    y = np.zeros(N)
    for B, t0, t1 in fir_level_taps(levels, taps):
        P = -(-(t1 - t0) // B)
        nb = -(-N // B)
        xp = np.concatenate([np.zeros(B), x, np.zeros(nb * B - N)])
        X = [np.fft.rfft(xp[j * B:(j + 2) * B]) for j in range(nb)]
        H = [np.fft.rfft(np.concatenate([h[t0 + p * B:min(t1, t0 + (p + 1) * B)], np.zeros(2 * B)])[:2 * B]) for p in range(P)]
        for m in range(nb):
            acc = np.zeros(B + 1, dtype=complex)
            for p in range(P):
                j = m - t0 // B - p
                if 0 <= j < nb:
                    acc = acc + X[j] * H[p]
            seg = np.fft.irfft(acc, 2 * B)[B:]
            y[m * B:min(N, (m + 1) * B)] += seg[:min(N, (m + 1) * B) - m * B]
    return ~np.isfinite(y)


def _levels(spec):
    return [{"B": B, "P": P} for B, P in spec]


FIR_MODELS = [  # (levels, taps): single levels with P = 1, 2, 5 and multi-level ladders as fir_schedule() draws them
    ([(8, 1)], 8), ([(8, 1)], 3), ([(8, 2)], 9), ([(8, 5)], 37), ([(16, 3)], 48),
    ([(4, 2), (8, 1)], 9), ([(4, 2), (8, 1), (16, 3)], 53), ([(8, 2), (16, 1), (32, 2)], 93),
]


@pytest.mark.parametrize("spec,taps", FIR_MODELS)
def test_fir_nan_window_against_a_blockwise_model(spec, taps):
    """The first non-finite frame of the model is fir_nan_window's first frame exactly (the start of the level-0 block
    holding n), and its last is before the window's end, for every n over several blocks and every latency offset."""
    levels = _levels(spec)
    Bl = spec[-1][0]
    for n in range(0, 4 * Bl):
        N = n + taps + 3 * Bl
        bad = np.nonzero(_fir_model(N, n, taps, levels))[0]
        lo, hi = fir_nan_window(n, taps, levels)
        assert bad[0] == lo and bad[-1] < hi, (spec, taps, n, bad[0], bad[-1], lo, hi)
        assert np.array_equal(bad, np.arange(bad[0], bad[-1] + 1)), (spec, n)
        lo2, hi2 = fir_nan_window(n, taps, levels, latency=17)
        assert (lo2, hi2) == (lo + 17, hi + 17)


def test_fir_b0_matches_the_plans_of_the_accuracy_cases():
    assert [fir_b0(h) for h in (0, 7, 64, 127, 128, 300, 1000, 2048, 4095, 4096, 32768)] == \
        [64, 64, 64, 64, 128, 256, 512, 2048, 2048, 4096, 8192]


def _rs_model(counts, n_, d, in_len, out_delay, Q, G):
    """The tiled kernel in numpy: per call, tiles of Q outputs from its first; a tile walks rows i_top down to i_bot
    in steps of 4 and every output multiplies every walked row with its tap (zero outside its window), as k_rs_poly and
    k_rs_mma(2) do.  Row n of input n is NaN, every other row zero.  Returns the non-finite outputs [input, output]."""
    total = int(np.sum(counts))
    ih = (out_delay + np.arange(total)) * d // n_
    rows_all = int(ih[-1]) + 1
    X = np.where(np.eye(rows_all, dtype=bool), np.nan, 0.0)   # X[r, n]: input n, row r
    bad = np.zeros((rows_all, total), dtype=bool)
    pos = 0
    for k in counts:
        for a in range(pos, pos + k, Q):
            b = min(a + Q, pos + k) - 1
            top, bot = ih[b], max(ih[a] - in_len + 1, 0)
            rows = np.array([top - j for j in range(4 * -(-(top - bot + 1) // 4)) if top - j >= 0])
            q = np.arange(a, b + 1)
            t = ih[q][:, None] - rows[None, :]
            ph = ((out_delay + q) * d % n_)[:, None]
            tap = np.where((t >= 0) & (t < in_len) & (rows[None, :] >= bot), G[ph, np.clip(t, 0, in_len - 1)], 0.0)
            y = np.einsum("qr,rn->nq", tap, X[rows])   # products in full: 0 x NaN stays NaN
            bad[:, a:b + 1] = ~np.isfinite(y)
        pos += k
    return bad


@pytest.mark.parametrize("n_,d,in_len,delay", [(3, 4, 10, 2), (4, 3, 9, 5), (1, 6, 13, 0), (6, 1, 7, 3), (5, 7, 11, 1)])
@pytest.mark.parametrize("Q", sorted({rs_expect_launch(4, tile, 1, 1)["Q"] for tile in range(1, 8)}) + [8])
def test_rs_nan_windows_against_a_tiled_model(n_, d, in_len, delay, Q):
    """Small rates, random non-zero taps, ragged calls (the drain is more calls): the tile mask equals the model's
    non-finite outputs for every input row n, and holds the exact window."""
    rng = np.random.default_rng(n_ * 100 + d)
    G = rng.uniform(0.5, 1.0, (n_, in_len))
    counts = [1, 0, 5, Q + 3, 2 * Q, 7, 3 * Q + 1]
    model = _rs_model(counts, n_, d, in_len, delay, Q, G)
    for n in range(model.shape[0]):
        exact, tile = rs_nan_windows(n, counts, n_, d, in_len, delay, Q)
        assert np.array_equal(tile, model[n]), (n, np.nonzero(tile)[0], np.nonzero(model[n])[0])
        assert not np.any(exact & ~tile), n
