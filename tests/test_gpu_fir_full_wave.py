"""GPU tier: the full-wave FIR plan against the exact convolution.

A single-level, direct-I/O plan whose fused kernel's CTAs outnumber half the SMs folds its tail ("full-wave").  From
2 * 8 + 3 partitions on its near tier has depth T = 8 (4 below), and with one tier it looks two blocks ahead instead of
three: the launch after block q covers the periods q+2+t with every partition p >= 2+t, and the fused kernel of block
j sums partitions 0 .. 1+t, 2 .. T+1 of them (all T+1 until a launch of the channel's class has covered j).  The
channel counts are computed from the device's SM count.

Every case runs the folded chain and the per-block MAC chain (DSP_B200_FIR_FOLD=0, T the same, look-ahead 3) on the same
input: whole aligned blocks from block 0 (start-up blocks included), then reset() and ragged calls.  Both must match
the exact convolution and each other.
"""
import zlib

import numpy as np
import pytest

from accuracy import dyadic_signal, exact_conv, fir_nerr
from test_gpu_accuracy import F2, F4, FIR_MAX, FIR_RMS, H_SHIFT, ir_family
from test_gpu_fir_fold import _run_form

pytestmark = pytest.mark.gpu


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def full_wave_channels(B):
    """The fewest channels, a multiple of 8, whose fused-kernel CTAs (one 4096-point or two 2048-point transforms each)
    outnumber half the SMs: 72 at 4096 frames and 136 at 2048 frames on 132 SMs."""
    cpb = 1 if B >= 4096 else 2
    C = 8
    while 2 * -(-C // cpb) <= _sms():
        C += 8
    return C


# name: (taps, block, plan fields)
FULL_WAVE_CASES = {
    "B4096_P18": (17 * F4 + 1, F4, dict(P=18, t_batch=4, stagger=0, class_width=1)),
    "B4096_P19": (18 * F4 + 1, F4, dict(P=19, t_batch=8, stagger=0, class_width=1)),
    "headline_B4096_P32": (131072, F4, dict(P=32, t_batch=8, stagger=1, class_width=4)),
    "B2048_P19": (18 * F2 + 1, F2, dict(P=19, t_batch=8, stagger=0, class_width=1)),
    "B2048_P26": (25 * F2 + 1, F2, dict(P=26, t_batch=8, stagger=1, class_width=4)),
}


@pytest.mark.parametrize("case", list(FULL_WAVE_CASES))
def test_fir_full_wave_matches_unfolded_and_exact(gpu_lib, case):
    """The full-wave plan reports its depth, lookahead = 2, l0_parts = T + 1, l0_parts_min = 2 and its class width; the
    per-block MAC form of the same shape keeps the depth with lookahead 3.  Both match the exact convolution and each
    other in whole blocks and ragged calls."""
    taps, B, want = FULL_WAVE_CASES[case]
    P, T = want["P"], want["t_batch"]
    C = full_wave_channels(B)
    N = (2 * P + 3) * B + 77
    rng = np.random.default_rng(zlib.crc32(b"full_wave" + case.encode()))
    h = ir_family("comb", taps, C, seed=taps + 2)
    x = dyadic_signal(rng, N, C)
    exact = exact_conv(x, h, H_SHIFT)
    nblk = N // B
    res = {fold: _run_form(gpu_lib, x, h, B, {}, fold) for fold in (True, False)}
    for fold, (whole, ragged, plan, launches, n_mac) in res.items():
        assert plan["levels"] == [{"B": B, "P": P}] and plan["tail_pf"] == 2 and plan["n_sel"] == C, (case, fold, plan)
        assert (plan["t_batch"], plan["t_far"], plan["stagger"]) == (T, 0, want["stagger"]), (case, fold, plan)
        if fold:
            assert (plan["lookahead"], plan["l0_parts"], plan["l0_parts_min"], plan["class_width"]) == (2, T + 1, 2, want["class_width"]), (case, plan)
        else:
            assert (plan["lookahead"], plan["l0_parts"], plan["l0_parts_min"], plan["class_width"]) == (3, 2, 2, 1), (case, plan)
        assert n_mac == (0 if fold else nblk), (case, fold, n_mac)
        for name, got, ref, xs in (("whole", whole, exact[:nblk * B], x[:nblk * B]), ("ragged", ragged, exact, x)):
            r, m = fir_nerr(got, ref, xs, h)
            assert r <= FIR_RMS and m <= FIR_MAX, (case, fold, name, r, m)
    if want["stagger"]:
        assert res[True][3] == 2 * nblk, (case, res[True][3])   # the fused kernel and one batch-tier class per block
    for name, i, n in (("whole", 0, nblk * B), ("ragged", 1, N)):
        r, m = fir_nerr(res[True][i], res[False][i], x[:n], h)
        assert r <= FIR_RMS and m <= FIR_MAX, (case, "folded vs unfolded", name, r, m)


def test_fir_full_wave_2048_frames_one_tier(gpu_lib):
    """131072 taps in 2048-frame blocks (64 partitions) at the full-wave count: one staggered tier of depth 8 with
    look-ahead 2 instead of tiers 4 + 8; a far tier asked for (16) keeps look-ahead 3."""
    from accuracy import env
    C = full_wave_channels(F2)
    h = np.zeros(131072)
    h[0] = 1.0
    for far, want in ((None, (8, 0, 1, 2, 9, 2)), ("16", (8, 16, 0, 3, 10, 3))):
        with env(DSP_B200_FIR_T2=far):
            ch = gpu_lib.Chain(48000, C).add_fir(h, block_hint=F2)
            plan = ch.describe()[0]
        ch.close()
        assert plan["levels"] == [{"B": F2, "P": 64}], plan
        got = tuple(plan[k] for k in ("t_batch", "t_far", "stagger", "lookahead", "l0_parts", "l0_parts_min"))
        assert got == want, (far, plan)


def test_fir_full_wave_threshold(gpu_lib):
    """Eight channels fewer than the full-wave count keep the plan of the smaller shapes: depth 4, look-ahead 3 (also
    with the fold forced), and the full-wave count itself takes depth 8 and look-ahead 2."""
    from accuracy import env
    C1 = full_wave_channels(F4)
    h = np.zeros(131072)
    h[0] = 1.0
    for C, fold, want in ((C1 - 8, None, (4, 3)), (C1 - 8, "1", (4, 3)), (C1, None, (8, 2))):
        with env(DSP_B200_FIR_FOLD=fold):
            ch = gpu_lib.Chain(48000, C).add_fir(h, block_hint=F4)
            plan = ch.describe()[0]
        ch.close()
        assert (plan["t_batch"], plan["lookahead"]) == want, (C, fold, plan)
        if fold or C == C1:
            assert (plan["l0_parts"], plan["l0_parts_min"]) == (want[0] + want[1] - 1, want[1]), (C, fold, plan)
