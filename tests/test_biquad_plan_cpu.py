"""CPU tier: the biquad cascade's host logic, dsp_b200/csrc/biquad_plan.h, compiled with g++ alone.

The scan table is checked for what it means, in numpy long double from the same double coefficients, not against a
restatement of the builder: T T^-1 = I; T sum_i G[i] s_i is the state the reference recurrence (biquad.h:79-81)
reaches after 16 samples from zero; T P[r] T^-1 is the zero-input map over 16 2^r samples; where eps is not clamped,
||P[r]||_2 <= 1.  bq_launch() (the kernel form, grid and launches of each call) against accuracy.bq_expect_launch,
which the GPU tests also check against describe().
"""
import ctypes

import numpy as np
import pytest

from accuracy import BQ_TBL, bq_expect_launch, header_lib

DRIVER = r"""
#include "biquad_plan.h"
#include <algorithm>
using namespace dspb200;
extern "C" {
// BQ_L, BQ_MAX_STAGES, BQ_NPOW, BQ_OFF_P, BQ_OFF_T, BQ_OFF_G, BQ_TBL
void layout(int *out)
{
	const int v[] = { BQ_L, BQ_MAX_STAGES, BQ_NPOW, BQ_OFF_P, BQ_OFF_T, BQ_OFF_G, BQ_TBL };
	std::copy(v, v + 7, out);
}
double eps_min() { return BQ_EPS_MIN; }
void stage_table(const double *cf, double *t) { bq_stage_table(cf, t); }
void table(int C, int S, const double *coefs, double *out)
{
	const std::vector<double> t = bq_table(C, S, coefs);
	std::copy(t.begin(), t.end(), out);
}
// ch, split, threads, grid, smem, span, launches
void launch(int C, int S, long frames, int force_ch, int force_split, long *out)
{
	const BqLaunch L = bq_launch(C, S, frames, force_ch, force_split);
	const long v[] = { L.ch, L.split, L.threads, L.grid, (long) L.smem, L.span, L.launches };
	std::copy(v, v + 7, out);
}
}
"""
L, NPOW = 16, 6
OFF_P, OFF_T, OFF_G = 6, 30, 38
U = 2.0 ** -53
LD = np.longdouble


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = header_lib(tmp_path_factory.mktemp("biquad_plan"), "biquadplan", DRIVER)
    dp = ctypes.POINTER(ctypes.c_double)
    lib.layout.argtypes = [ctypes.POINTER(ctypes.c_int)]
    lib.eps_min.restype = ctypes.c_double
    lib.stage_table.argtypes = [dp, dp]
    lib.table.argtypes = [ctypes.c_int, ctypes.c_int, dp, dp]
    lib.launch.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_long)]
    return lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def stage_tables(lib, coefs):
    """[N, BQ_TBL] tables of the sections coefs [N, 5]."""
    coefs = np.ascontiguousarray(coefs, dtype=np.float64)
    out = np.zeros((len(coefs), BQ_TBL))
    for k in range(len(coefs)):
        lib.stage_table(_ptr(coefs[k]), _ptr(out[k]))
    return out


# ------------------------------------------------------------------------------------------------------------
# sections
# ------------------------------------------------------------------------------------------------------------
def cookbook(kind, fs, f0, q):
    """The audio EQ cookbook's lowpass / highpass / notch, normalised to c0..c4 (b0, b1, b2, a1, a2 over a0)."""
    w = 2 * np.pi * f0 / fs
    cw, al = np.cos(w), np.sin(w) / (2 * q)
    b = {"lowpass": ((1 - cw) / 2, 1 - cw, (1 - cw) / 2), "highpass": ((1 + cw) / 2, -(1 + cw), (1 + cw) / 2),
         "notch": (1.0, -2 * cw, 1.0)}[kind]
    a0 = 1 + al
    return [b[0] / a0, b[1] / a0, b[2] / a0, -2 * cw / a0, (1 - al) / a0]


def sections(n_random=64, seed=5):
    """name -> c0..c4: the low-corner sections of the GPU accuracy tests, a double pole, complex poles, first-order
    sections, the identity, and seeded random stable sections with real or complex poles."""
    s = {
        "lowpass_10_192k_q5": cookbook("lowpass", 192000, 10.0, 5.0),
        "lowpass_10_192k": cookbook("lowpass", 192000, 10.0, 0.707),
        "highpass_10_192k_q10": cookbook("highpass", 192000, 10.0, 10.0),
        "notch_10_192k_q10": cookbook("notch", 192000, 10.0, 10.0),
        "highpass_5_44k_q0.5": cookbook("highpass", 44100, 5.0, 0.5),
        "lowpass_80_48k": cookbook("lowpass", 48000, 80.0, 0.707),
        "lowpass_8k_48k": cookbook("lowpass", 48000, 8000.0, 0.707),
        "double_pole_0.999": [0.25, 0.5, 0.25, -1.998, 0.999 * 0.999],
        "double_pole_-0.5": [1.0, 0.0, 0.0, 1.0, 0.25],
        "complex_0.9_1rad": [0.3, -0.1, 0.2, -2 * 0.9 * np.cos(1.0), 0.81],
        "complex_0.99999_3rad": [1.0, 1.0, 1.0, -2 * 0.99999 * np.cos(3.0), 0.99999 ** 2],
        "first_order_lowpass": [0.5 * (1 - 0.9987), 0.5 * (1 - 0.9987), 0.0, -0.9987, 0.0],
        "first_order_allpass": [-0.6, 1.0, 0.0, -0.6, 0.0],
        "identity": [1.0, 0.0, 0.0, 0.0, 0.0],
    }
    rng = np.random.default_rng(seed)
    for k in range(n_random):
        if k % 2:
            p1, p2 = rng.uniform(-0.9999, 0.9999, 2)
            a1, a2 = -(p1 + p2), p1 * p2
        else:
            r, th = rng.uniform(0.0, 0.9999), rng.uniform(0.0, np.pi)
            a1, a2 = -2 * r * np.cos(th), r * r
        s["random_%d" % k] = [*rng.uniform(-2, 2, 3), a1, a2]
    return s


SECTIONS = sections()


def _unpack(t):
    """(T, T^-1, P [NPOW, 2, 2], G [L, 2]) of tables t [N, BQ_TBL], in long double."""
    t = t.astype(LD)
    return (t[:, OFF_T:OFF_T + 4].reshape(-1, 2, 2), t[:, OFF_T + 4:OFF_T + 8].reshape(-1, 2, 2),
            t[:, OFF_P:OFF_P + 4 * NPOW].reshape(-1, NPOW, 2, 2), t[:, OFF_G:OFF_G + 2 * L].reshape(-1, L, 2))


# ------------------------------------------------------------------------------------------------------------
# layout
# ------------------------------------------------------------------------------------------------------------
def test_layout(lib):
    """The table's pieces start on 16-byte boundaries, the [C][S] table is the per-stage table of coefs[s][c], and its
    entries 0-4 are that section's coefficients bit for bit (5 is a zero pad)."""
    lay = (ctypes.c_int * 7)()
    lib.layout(lay)
    assert list(lay) == [L, 16, NPOW, OFF_P, OFF_T, OFF_G, BQ_TBL]
    assert all(v % 2 == 0 for v in (OFF_P, OFF_T, OFF_G, BQ_TBL))
    assert lib.eps_min() == 1.0 / 32
    rng = np.random.default_rng(1)
    pool = np.array(list(SECTIONS.values()))
    for C, S in ((1, 1), (3, 4), (5, 16)):
        coefs = np.ascontiguousarray(pool[rng.integers(0, len(pool), S * C)].reshape(S, C, 5))
        got = np.zeros(C * S * BQ_TBL)
        lib.table(C, S, _ptr(coefs), _ptr(got))
        got = got.reshape(C, S, BQ_TBL)
        want = stage_tables(lib, coefs.transpose(1, 0, 2).reshape(-1, 5)).reshape(C, S, BQ_TBL)
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (C, S)
        assert np.array_equal(got[:, :, :5].view(np.uint64), coefs.transpose(1, 0, 2).view(np.uint64))
        assert not got[:, :, 5].any()


# ------------------------------------------------------------------------------------------------------------
# what the table means
# ------------------------------------------------------------------------------------------------------------
# Tolerances in units of u = 2^-53 of each check's scale.  Largest errors measured (x86-64, g++ with 80-bit long double)
# on SECTIONS, and in brackets on 10,000 further random sections: T T^-1 - I 1.3 (1.4); the chunk's end state 0.9 (1.5);
# ||P[r]||_2 <= 1 everywhere.  The zero-input maps reach 24 (600) on nearly double complex poles, where the builder's
# long-double M = T^-1 A T loses bits in (alpha^2 - c4) / eps and its 16 2^r-fold powers amplify that; 8.7 on the
# cookbook and double-pole sections, and 4.2 on the sections of SECTIONS whose eps is not clamped.
TOL_INV, TOL_END, TOL_MAP, TOL_NORM = 3, 4, 64, 4


@pytest.fixture(scope="module")
def tables(lib):
    coefs = np.array(list(SECTIONS.values()))
    return coefs, stage_tables(lib, coefs)


def _clamped(coefs):
    c = coefs.astype(LD)
    return np.sqrt(np.abs(c[:, 3] ** 2 / 4 - c[:, 4])) < LD(1) / 32


def test_eps_clamp(tables):
    """The basis T = [[1, 0], [-alpha, eps]]: eps = sqrt|alpha^2 - c4|, clamped to 1/32 for (near-)double poles --
    the double poles, the identity and the 10 Hz sections among them -- and T[3] is then 1/32 exactly."""
    coefs, t = tables
    T = t[:, OFF_T:OFF_T + 4]
    clamped = _clamped(coefs)
    names = list(SECTIONS)
    for k in ("double_pole_0.999", "double_pole_-0.5", "identity", "lowpass_10_192k_q5", "highpass_10_192k_q10"):
        assert clamped[names.index(k)], k
    for k in ("complex_0.9_1rad", "first_order_lowpass", "lowpass_8k_48k"):
        assert not clamped[names.index(k)], k
    assert np.all(T[clamped, 3] == 1.0 / 32)
    assert np.all(T[~clamped, 3] >= 1.0 / 32)
    assert np.array_equal(T[:, 0], np.ones(len(T))) and not T[:, 1].any()
    assert np.array_equal(T[:, 2], coefs[:, 3] / 2)   # -alpha = c3 / 2, exact


def _err(name, got, want, scale, tol):
    """max |got - want| / (u scale) over everything (where the scale is 0, got must equal want), asserted <= tol;
    returns the worst ratio."""
    d = np.abs(got - want)
    d = np.divide(d, U * scale, out=np.where(d == 0, 0, np.inf).astype(LD), where=scale > 0)
    r = np.max(d, axis=tuple(range(1, got.ndim)))
    worst = int(np.argmax(r))
    assert r[worst] <= tol, (name, list(SECTIONS)[worst], float(r[worst]))
    return float(r[worst])


def test_basis_inverse(tables):
    """T T^-1 = I, to rounding of the entries."""
    _, t = tables
    T, Ti, _, _ = _unpack(t)
    _err("T Ti", T @ Ti, np.eye(2, dtype=LD), np.abs(T) @ np.abs(Ti), TOL_INV)


def test_chunk_end_state(tables):
    """T sum_i G[i] s_i equals the end state of the reference recurrence run over the chunk s_0..s_15 from a zero state
    (long double), for three seeded chunks per section."""
    coefs, t = tables
    T, _, _, G = _unpack(t)
    c = coefs.astype(LD)
    Ak = [np.broadcast_to(np.eye(2, dtype=LD), (len(c), 2, 2))]
    for _ in range(L - 1):   # A^k: the zero-input step (m0, m1) -> (m1 - c3 m0, -c4 m0) on the columns
        Ak.append(np.stack([Ak[-1][:, 1] - c[:, 3, None] * Ak[-1][:, 0], -c[:, 4, None] * Ak[-1][:, 0]], axis=1))
    Ak = np.stack(Ak[::-1], axis=1)   # [n, i]: A^(L-1-i)
    Bmag = np.stack([np.abs(c[:, 1]) + np.abs(c[:, 3] * c[:, 0]), np.abs(c[:, 2]) + np.abs(c[:, 4] * c[:, 0])], axis=1)
    rng = np.random.default_rng(2)
    for _ in range(3):
        s = rng.uniform(-1, 1, (len(c), L)).astype(LD)
        m0, m1 = np.zeros(len(c), dtype=LD), np.zeros(len(c), dtype=LD)
        for i in range(L):
            r = c[:, 0] * s[:, i] + m0
            m0, m1 = m1 + c[:, 1] * s[:, i] - c[:, 3] * r, c[:, 2] * s[:, i] - c[:, 4] * r
        got = np.einsum("nab,nb->na", T, np.einsum("nij,ni->nj", G, s))
        # the stored entries' rounding, plus the long-double rounding of B's terms (A^(L-1-i) |B| |s_i| 2^-64), which
        # cancel to a small B = (c1 - c3 c0, c2 - c4 c0) in low-corner sections, in the builder and in the recurrence
        scale = (np.einsum("nab,nib,ni->na", np.abs(T), np.abs(G), np.abs(s))
                 + 2.0 ** -11 * np.einsum("niab,nb,ni->na", np.abs(Ak), Bmag, np.abs(s)))
        _err("end state", got, np.stack([m0, m1], axis=1), scale, TOL_END)


def test_zero_input_maps(tables):
    """T P[r] T^-1 equals A^(16 2^r), the zero-input map over 16 2^r samples (the recurrence stepped in long double from
    the two unit states), r = 0..5."""
    coefs, t = tables
    T, Ti, P, _ = _unpack(t)
    c = coefs.astype(LD)
    Z = np.broadcast_to(np.eye(2, dtype=LD), (len(c), 2, 2)).copy()   # columns: the two states
    for k in range(1, (L << (NPOW - 1)) + 1):
        r = Z[:, 0]
        Z = np.stack([Z[:, 1] - c[:, 3, None] * r, -c[:, 4, None] * r], axis=1)
        if k % L == 0 and (k // L) & (k // L - 1) == 0:
            j = (k // L).bit_length() - 1
            # (2^-1000: entries that underflow in double, long decayed in long double)
            _err("map %d" % k, T @ P[:, j] @ Ti, Z, np.abs(T) @ np.abs(P[:, j]) @ np.abs(Ti) + 2.0 ** -1000 / U, TOL_MAP)


def test_powers_bounded(tables):
    """Where eps is not clamped, M is normal and its powers P[r] have spectral norm at most 1 (the poles are inside the
    unit circle): the property the basis exists for."""
    coefs, t = tables
    _, _, P, _ = _unpack(t)
    keep = ~_clamped(coefs)
    assert keep.sum() > len(SECTIONS) // 2
    norms = np.linalg.norm(P[keep].astype(np.float64), ord=2, axis=(2, 3))
    assert np.max(norms) <= 1 + TOL_NORM * U, float((np.max(norms) - 1) / U)


# ------------------------------------------------------------------------------------------------------------
# launch policy
# ------------------------------------------------------------------------------------------------------------
def test_launch(lib):
    """bq_launch() against bq_expect_launch, field by field, on frames around the split threshold and the tiles,
    every DSP_B200_BQ_CH and DSP_B200_BQ_SPLIT case (unset, off, on, other values), and channel counts that leave a
    partial last CTA."""
    out = (ctypes.c_long * 7)()
    keys = ("ch", "split", "threads", "grid", "smem", "span", "launches")
    seen = set()
    for frames in (1, 2047, 2048, 2049, 4096, 4097, 8192, 12289):
        for fc in (None, 0, 1, 2, 3, 4, -1, 8):
            for fsp in (None, 0, 1, 2):
                for C in (1, 2, 3, 4, 5, 256, 257):
                    for S in (1, 16):
                        lib.launch(C, S, frames, 0 if fc is None else fc, -1 if fsp is None else fsp, out)
                        got = dict(zip(keys, out))
                        want = bq_expect_launch(C, S, frames, fc, fsp)
                        assert got == want, (frames, fc, fsp, C, S, got, want)
                        seen.add((got["ch"], got["split"]))
    assert seen == {(1, 0), (2, 0), (2, 1), (4, 0)}, seen


def test_launch_shared_memory_fits_default(lib):
    """No launch asks for more than the 48 KB of dynamic shared memory a kernel gets without cudaFuncSetAttribute."""
    out = (ctypes.c_long * 7)()
    for S in range(1, 17):
        for fc in (0, 1, 4):
            for fsp in (-1, 0, 1):
                lib.launch(257, S, 4096, fc, fsp, out)
                assert out[4] <= 48 * 1024, (S, fc, fsp, out[4])
