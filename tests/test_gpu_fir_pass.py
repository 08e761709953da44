"""GPU tier: the mid-window pass of the full-wave FIR plan against the exact convolution.

On a staggered full-wave plan with one near tier of depth T and look-ahead 2, the grid launched after block q' also
adds, for the class whose tier launch came after block q = q' - m, partitions 2+t-m .. 1+t to the periods q+2+t with
t >= m.  The fused kernel then sums 0 .. 1+t for t < m and 0 .. 1+t-m from t = m on: at most 1 + max(m, T - m)
partitions once every class has had its pass, instead of T + 1.  The channel counts are computed from the device's SM
count.

Every case runs the pass form and DSP_B200_FIR_PASS=0 on the same input: whole aligned blocks from block 0 (start-up
blocks included), then reset() and ragged calls.  Both must match the exact convolution and each other, and both
launch two kernels per block.
"""
import zlib

import numpy as np
import pytest

from accuracy import PASS_CASES, dyadic_signal, exact_conv, fir_nerr
from test_gpu_accuracy import F2, F4, FIR_MAX, FIR_RMS, H_SHIFT, ir_family
from test_gpu_fir_fold import _run_form
from test_gpu_fir_full_wave import full_wave_channels

pytestmark = pytest.mark.gpu

_inputs = {}


def _case_input(taps, B, P, envs):
    """(x, h, exact, pass-less run) of a shape, shared by the cases that differ only in the pass depth."""
    key = (taps, B, P, tuple(sorted(envs.items())))
    if key not in _inputs:
        C = full_wave_channels(B)
        N = (2 * P + 3) * B + 77
        rng = np.random.default_rng(zlib.crc32(b"fir_pass%d_%d" % (taps, B)))
        h = ir_family("comb", taps, C, seed=taps + 3)
        x = dyadic_signal(rng, N, C)
        exact = exact_conv(x, h, H_SHIFT)
        _inputs.clear()
        _inputs[key] = (x, h, exact, None)
    return key


@pytest.mark.parametrize("case", list(PASS_CASES))
def test_fir_pass_matches_passless_and_exact(gpu_lib, case):
    """The pass form reports pass_m, l0_parts = T + 1 (start-up), l0_parts_min = 2 and l0_parts_steady = 1 + max(m, T -
    m); DSP_B200_FIR_PASS=0 reports pass_m = 0 and l0_parts_steady = T + 1.  Both launch the fused kernel and one
    batch grid per block and match the exact convolution and each other in whole blocks and ragged calls."""
    taps, B, P, envs, T, m = PASS_CASES[case]
    key = _case_input(taps, B, P, envs)
    x, h, exact, nopass = _inputs[key]
    if nopass is None:
        nopass = _run_form(gpu_lib, x, h, B, dict(envs, DSP_B200_FIR_PASS=0), True)
        _inputs[key] = (x, h, exact, nopass)
    withpass = _run_form(gpu_lib, x, h, B, dict(envs, DSP_B200_FIR_PASS=m), True)
    N = x.shape[0]
    nblk = N // B
    want_m = T // 2 if m is None else m
    for mm, (whole, ragged, plan, launches, n_mac) in ((want_m, withpass), (0, nopass)):
        assert plan["levels"] == [{"B": B, "P": P}] and plan["tail_pf"] == 2, (case, mm, plan)
        assert (plan["t_batch"], plan["t_far"], plan["stagger"], plan["class_width"], plan["lookahead"]) == (T, 0, 1, 4, 2), (case, mm, plan)
        steady = 1 + max(mm, T - mm) if mm else T + 1
        assert (plan["pass_m"], plan["l0_parts"], plan["l0_parts_min"], plan["l0_parts_steady"]) == (mm, T + 1, 2, steady), (case, plan)
        assert n_mac == 0 and launches == 2 * nblk, (case, mm, n_mac, launches)
        for name, got, ref, xs in (("whole", whole, exact[:nblk * B], x[:nblk * B]), ("ragged", ragged, exact, x)):
            r, mx = fir_nerr(got, ref, xs, h)
            assert r <= FIR_RMS and mx <= FIR_MAX, (case, mm, name, r, mx)
    for name, i, n in (("whole", 0, nblk * B), ("ragged", 1, N)):
        r, mx = fir_nerr(withpass[i], nopass[i], x[:n], h)
        assert r <= FIR_RMS and mx <= FIR_MAX, (case, "pass vs pass-less", name, r, mx)


def test_fir_pass_only_on_lookahead_2(gpu_lib):
    """Plans without a staggered single tier at look-ahead 2 take no pass: the per-block MAC form, a far tier, and a
    channel count below the full-wave threshold."""
    from accuracy import env
    h = np.zeros(131072)
    h[0] = 1.0
    for C, B, envs in ((full_wave_channels(F4), F4, dict(DSP_B200_FIR_FOLD=0)),
                       (full_wave_channels(F2), F2, dict(DSP_B200_FIR_T2=16)),
                       (full_wave_channels(F4) - 8, F4, {})):
        with env(**envs):
            ch = gpu_lib.Chain(48000, C).add_fir(h, block_hint=B)
            plan = ch.describe()[0]
        ch.close()
        assert plan["pass_m"] == 0 and plan["l0_parts_steady"] == plan["l0_parts"], (C, B, envs, plan)
