"""GPU tier: the folded FIR tail with the near tier's triangle against the exact convolution.

Folded, the near-tier launch after block q covers the periods j = q+3+t (t < T) with every partition p >= 3+t, and
the fused kernel of block j sums partitions 0 .. 2+t of each channel: 3 .. T+2 of them, by the channel's class and
the block.  Until a class has had its first launch covering j, its channels sum all T+2.  Staggered classes are groups
of describe() "class_width" adjacent channels (min(4, channels / T), a power of two).

Every case runs the folded chain (DSP_B200_FIR_FOLD=1) and the per-block MAC chain (=0) on the same input: whole
aligned blocks from block 0 (the start-up blocks whose classes no launch has covered yet included), then reset() and
ragged calls.  Both must match the exact convolution and each other.
"""
import zlib

import numpy as np
import pytest

from accuracy import dyadic_signal, exact_conv, fir_nerr
from test_gpu_accuracy import F2, F4, FIR_MAX, FIR_RMS, H_SHIFT, ir_family
from test_gpu_fir_fold import _run_form

pytestmark = pytest.mark.gpu

# name: (taps, channels, block, envs, plan fields)
TRIANGLE_CASES = {
    "headline_8ch": (131072, 8, F4, {}, dict(P=32, t_batch=4, t_far=0, stagger=1, class_width=2)),
    "headline_32ch": (131072, 32, F4, {}, dict(P=32, t_batch=4, t_far=0, stagger=1, class_width=4)),
    # 2048-point transforms, two channels per CTA in different classes: the CTA's two transform groups sum different counts
    "B2048_P22_stagger": (21 * F2 + 1, 4, F2, {}, dict(P=22, t_batch=4, t_far=0, stagger=1, class_width=1)),
    "B2048_P11_whole": (10 * F2 + 1, 4, F2, {}, dict(P=11, t_batch=4, t_far=0, stagger=0, class_width=1)),
    "B2048_P48_far": (47 * F2 + 1, 4, F2, {}, dict(P=48, t_batch=4, t_far=8, stagger=0, class_width=1)),
    "B2048_P24_T6": (23 * F2 + 1, 12, F2, dict(DSP_B200_FIR_T="6"), dict(P=24, t_batch=6, t_far=0, stagger=1, class_width=2)),
    "B2048_P26_T8": (25 * F2 + 1, 8, F2, dict(DSP_B200_FIR_T="8"), dict(P=26, t_batch=8, t_far=0, stagger=1, class_width=1)),
}


@pytest.mark.parametrize("case", list(TRIANGLE_CASES))
def test_fir_triangle_matches_unfolded_and_exact(gpu_lib, case):
    """The folded chain reports l0_parts = T+2, l0_parts_min = 3 and its class width, launches two kernels per block
    when staggered, and matches the exact convolution and the per-block MAC chain in whole blocks and ragged calls."""
    taps, C, B, envs, want = TRIANGLE_CASES[case]
    P, T = want["P"], want["t_batch"]
    N = (2 * P + 3) * B + 77
    rng = np.random.default_rng(zlib.crc32(b"triangle" + case.encode()))
    h = ir_family("comb", taps, C, seed=taps + 1)
    x = dyadic_signal(rng, N, C)
    exact = exact_conv(x, h, H_SHIFT)
    nblk = N // B
    res = {fold: _run_form(gpu_lib, x, h, B, envs, fold) for fold in (True, False)}
    for fold, (whole, ragged, plan, launches, n_mac) in res.items():
        assert plan["levels"] == [{"B": B, "P": P}] and plan["tail_pf"] == 2, (case, fold, plan)
        for k in ("t_batch", "t_far", "stagger"):
            assert plan[k] == want[k], (case, fold, k, plan)
        if fold:
            assert (plan["l0_parts"], plan["l0_parts_min"], plan["class_width"]) == (T + 2, 3, want["class_width"]), (case, plan)
        else:
            assert (plan["l0_parts"], plan["l0_parts_min"], plan["class_width"]) == (2, 2, 1), (case, plan)
        assert n_mac == (0 if fold else nblk), (case, fold, n_mac)
        for name, got, ref, xs in (("whole", whole, exact[:nblk * B], x[:nblk * B]), ("ragged", ragged, exact, x)):
            r, m = fir_nerr(got, ref, xs, h)
            assert r <= FIR_RMS and m <= FIR_MAX, (case, fold, name, r, m)
    if want["stagger"]:
        assert res[True][3] == 2 * nblk, (case, res[True][3])   # the fused kernel and one batch-tier class per block
    for name, i, n in (("whole", 0, nblk * B), ("ragged", 1, N)):
        r, m = fir_nerr(res[True][i], res[False][i], x[:n], h)
        assert r <= FIR_RMS and m <= FIR_MAX, (case, "folded vs unfolded", name, r, m)
