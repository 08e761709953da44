"""GPU tier: the folded FIR tail against the exact convolution.

On single-level plans with a batch tier the fused kernel sums partitions 0 .. t_batch+1 itself and starts from the
batch tier's V_j ("folded"; the default when its CTAs outnumber half the SMs, DSP_B200_FIR_FOLD=1 here); with
DSP_B200_FIR_FOLD=0 the per-block MAC k_fir_mac sums partitions 2 .. t_batch+1 a block period ahead.  Both forms run the same stream -- whole aligned blocks through
run_device (the cluster form, the high-priority stream), then reset() and ragged calls (the general path mixed with
the fused kernel) -- and must match the exact convolution and each other.
"""
import zlib

import numpy as np
import pytest

from accuracy import FOLD_CASES, dyadic_signal, env, exact_conv, fir_nerr
from test_gpu_accuracy import FIR_MAX, FIR_RMS, H_SHIFT, _ragged_sizes, _run_sizes, ir_family

pytestmark = pytest.mark.gpu

def _run_form(gpu_lib, x, h, B, envs, fold):
    """Whole blocks through run_device, then reset() and ragged calls; -> (whole, ragged, plan, launches, fir_mac
    launches of the whole-block pass)."""
    import torch
    N, C = x.shape
    nblk = N // B
    rng = np.random.default_rng(zlib.crc32(b"fold%d" % N))
    with env(DSP_B200_FIR_FOLD="1" if fold else "0", **envs):
        ch = gpu_lib.Chain(48000, C).add_fir(h, block_hint=B)
        st = torch.cuda.current_stream().cuda_stream
        d_x = torch.from_numpy(np.ascontiguousarray(x[:nblk * B]).reshape(-1)).cuda()
        d_y = torch.zeros_like(d_x)
        torch.cuda.synchronize()
        gpu_lib.profile_read("fir_mac")
        gpu_lib.profile_enable(True)
        l0 = gpu_lib.kernel_launches()
        for b in range(nblk):
            off = 8 * b * B * C
            assert ch.run_device(0, B, d_x.data_ptr() + off, d_y.data_ptr() + off, st) == B
        launches = gpu_lib.kernel_launches() - l0
        ch.join(0, st)
        torch.cuda.synchronize()
        gpu_lib.profile_enable(False)
        _, n_mac = gpu_lib.profile_read("fir_mac")
        whole = d_y.cpu().numpy().reshape(nblk * B, C)
        ch.reset()
        ragged = _run_sizes(ch, x, _ragged_sizes(rng, N, B))
        plan = ch.describe()[0]
    ch.close()
    return whole, ragged, plan, launches, n_mac


@pytest.mark.parametrize("case", list(FOLD_CASES))
def test_fir_fold_matches_unfolded_and_exact(gpu_lib, case):
    """Folded and unfolded chains on the same input: both within the exact-convolution bounds, in whole blocks and in
    ragged calls; the folded plan reports l0_parts = t_batch + 2 and launches no k_fir_mac (one launch per block less
    than the unfolded form, which launches one k_fir_mac per block)."""
    taps, C, B, envs, want = FOLD_CASES[case]
    P = want["P"]
    N = (2 * P + 3) * B + 77
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    h = ir_family("comb", taps, C, seed=taps)
    x = dyadic_signal(rng, N, C)
    exact = exact_conv(x, h, H_SHIFT)
    nblk = N // B
    res = {fold: _run_form(gpu_lib, x, h, B, envs, fold) for fold in (True, False)}
    for fold, (whole, ragged, plan, launches, n_mac) in res.items():
        assert plan["levels"] == [{"B": B, "P": P}] and plan["tail_pf"] == 2, (case, fold, plan)
        for k in ("t_batch", "t_far", "stagger"):
            assert plan[k] == want[k], (case, fold, k, plan)
        assert plan["l0_parts"] == (want["t_batch"] + 2 if fold else 2), (case, fold, plan)
        assert n_mac == (0 if fold else nblk), (case, fold, n_mac)
        for name, got, ref, xs in (("whole", whole, exact[:nblk * B], x[:nblk * B]), ("ragged", ragged, exact, x)):
            r, m = fir_nerr(got, ref, xs, h)
            assert r <= FIR_RMS and m <= FIR_MAX, (case, fold, name, r, m)
    assert res[True][3] == res[False][3] - nblk, (case, res[True][3], res[False][3])
    if want["stagger"]:
        assert res[True][3] == 2 * nblk, (case, res[True][3])   # the fused kernel and one batch-tier class per block
    r, m = fir_nerr(res[True][0], res[False][0], x[:nblk * B], h)
    assert r <= FIR_RMS and m <= FIR_MAX, (case, "folded vs unfolded", r, m)
