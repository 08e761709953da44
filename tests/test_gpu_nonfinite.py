"""GPU tier: NaN and Inf samples stay in their channel and in the frames that depend on them, and reset() forgets them.

Every case runs one stream twice, on two fresh chains: clean (sample n of channel k is 0.0) and poisoned (that sample
is NaN, +Inf or -Inf, several (k, n) pairs per stream on different channels).  No kernel uses atomics, so:
  1. isolation: every channel that was not poisoned is bit-identical between the two runs (pair, cluster and tile
     partners of a poisoned channel, other slabs of a sharded chain);
  2. causality: every output that cannot depend on input n is bit-identical -- gain and align: all but frame
     n + d_k; biquad: every frame before n; FIR: every frame before the level-0 block holding n (+ latency)
     (accuracy.fir_nan_window); resample: every output whose CTA tile does not read input row n
     (accuracy.rs_nan_windows);
  3. extent: biquad -- from n on, non-finite exactly where the reference's own FP64 recurrence is
     (restate.biquad_cascade): to the end of the stream; FIR -- every frame from n + taps + 2 B_last (+ latency) on is
     finite and bit-identical; resample -- every output outside the tiles that read row n; gain and align -- exactly one
     non-finite frame (none when align discards it);
  4. reset(): the poisoned chain, reset and fed the clean stream, gives a fresh chain's clean output bit for bit.

Bounds (derived in tests/accuracy.py next to each helper).  The resampler's bound is its tile, not its exact window:
a CTA multiplies every input row it walks with every one of its Q outputs' taps, zero where the row is outside an
output's window, so a NaN reaches up to Q - 1 outputs before the first output whose window holds it (and a few after
the last).  The reference does the same on a larger scale (its FFT block of in_len frames), so this is the kernel's
granularity, not a fault; tightening it would mean a tap-window test per product in the hot loop.

Measured on an H100 80GB HBM3 (700 W limit): isolation and reset() hold bit for bit everywhere.  Biquad: non-finite
from n to the end exactly where the FP64 recurrence is, on every form and knob.  Gain and align: one frame.  Resample:
the tile bound holds with no margin (it is exact); the NaN reached up to 62 outputs before its exact window and 66 after
it.  FIR (multi-level at 64 frames, the pipeline kernel at 4096, the fused, latency, multi-level
and selector edges, the re-plan): the first differing frame is the level-0 block's first (no margin, as derived) and the
last is within the bound.  FIR with a batch tier, and the bulk form: the same, once the kernel fix described in
test_fir_plan_paths_nonfinite was made (over all FIR cases the end margin is 1 to 9039 frames).  Margins of each case are appended
as JSON lines to the file DSP_B200_ACCURACY_LOG names, when it is set.
"""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

from accuracy import (FIR_CASES, FIR_EDGES, bq_expect_launch, dyadic_signal, env, fir_b0, fir_nan_window, rs_expect_launch,
                      rs_nan_windows)
from test_gpu_accuracy import (BQ_CASCADE, BQ_SECTIONS, RS_SHAPES, _drain, _ragged_sizes, _record,
                               _run_calls, _rs_chain, ir_family, rs_bases, _tiled)

pytestmark = pytest.mark.gpu
POISON = (np.nan, np.inf, -np.inf)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------
# the pattern
# ------------------------------------------------------------------------------------------------------------
def _poisoned(x, poisons):
    """(clean, poisoned) copies of x: sample n of channel k is 0.0, resp. NaN / +Inf / -Inf in turn."""
    clean = np.array(x, dtype=np.float64, copy=True)
    bad = clean.copy()
    for i, (k, n) in enumerate(poisons):
        clean[n, k] = 0.0
        bad[n, k] = POISON[i % 3]
    return clean, bad


def _same_calls(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        if g is None or w is None:
            assert g is None and w is None, (what, i)
            continue
        assert g.shape == w.shape and np.array_equal(g, w), (what, "call", i, "differs from a fresh chain's clean output")


def _twice(make, x, poisons, run, envs=None, fresh=True):
    """Clean and poisoned runs of `run(chain, x) -> [outputs per call]` on fresh chains from make(); the poisoned chain
    is then reset and fed the clean stream, which must give the clean run's outputs bit for bit.  fresh=False where
    reset() keeps state that a fresh chain does not have (the plan after re-planning, the resampler's drain counters):
    the clean chain is reset and run again too, and the two must agree.  Returns (clean outputs, poisoned outputs,
    describe() of the poisoned chain before the reset)."""
    clean, bad = _poisoned(x, poisons)
    with env(**(envs or {})):
        a = make()
        want = run(a, clean)
        if not fresh:
            a.reset()
            want_again = run(a, clean)
        a.close()
        b = make()
        got = run(b, bad)
        plan = b.describe()
        b.reset()
        again = run(b, clean)
        b.close()
    _same_calls(again, want if fresh else want_again, "after reset()")
    return want, got, plan


def _cat(outs, C):
    outs = [o for o in outs if o is not None]
    return np.concatenate(outs) if outs else np.zeros((0, C))


def _isolated(want, got, poisons, what):
    ks = {k for k, _ in poisons}
    assert want.shape == got.shape, (what, want.shape, got.shape)
    for c in range(want.shape[1]):
        if c not in ks:
            assert np.array_equal(got[:, c], want[:, c]), (what, "channel", c, "changed by a non-finite sample elsewhere")


def _differs(want, got):
    """Frames where got is not bit-identical to want (NaN never equals anything)."""
    return ~((got == want) | (np.isnan(got) & np.isnan(want)))


# ------------------------------------------------------------------------------------------------------------
# FIR
# ------------------------------------------------------------------------------------------------------------
def _fir_poisons(sizes, B0, chans):
    """One position per channel: the middle of a call that spans several level-0 blocks (in its second block), the
    first and the last frame of a call, and the first and last frame of a level-0 block (n = 0, -1 mod B0) -- those
    first when the calls are not whole blocks.  Calls from the third on."""
    starts = np.concatenate([[0], np.cumsum(sizes)])
    i = next((j for j in range(2, min(len(sizes), 40)) if sizes[j] >= 2 * B0), 2)
    mid = int(starts[i]) + (B0 + B0 // 2 if sizes[i] >= 2 * B0 else sizes[i] // 2)
    first = int(starts[3])
    last = int(starts[5]) - 1
    b = (int(starts[4]) // B0 + 2) * B0
    part = [b, b + 3 * B0 - 1]
    pos = [mid, first, last] + part if all(s % B0 == 0 for s in sizes[:6]) else [mid] + part + [first, last]
    return list(zip(chans, pos))


def _fir_check(name, want, got, poisons, taps, plan, latency=0, sel=None):
    """Isolation, causality and extent per poisoned channel; unselected channels pass the sample through at n."""
    _isolated(want, got, poisons, name)
    for k, n in poisons:
        diff = np.nonzero(_differs(want[:, k], got[:, k]))[0]
        if sel is not None and not sel[k]:
            assert diff.tolist() == [n] and not np.isfinite(got[n, k]), (name, k, n, diff[:8])
            continue
        lo, hi = fir_nan_window(n, taps, plan["levels"], latency)
        assert hi <= got.shape[0], (name, "stream too short for the extent bound", hi, got.shape[0])
        assert not np.isfinite(got[n + latency, k]), (name, k, n, "the sample never reached the output")
        assert diff[0] >= lo, (name, k, n, "differs at frame %d, before the level-0 block's start %d" % (diff[0], lo))
        assert diff[-1] < hi, (name, k, n, "still differs at frame %d, bound %d" % (diff[-1], hi))
        assert np.all(np.isfinite(got[hi:, k])), (name, k, n)
        _record("nonfinite", name, op="fir", k=k, n=n, first_margin=int(diff[0] - lo), end_margin=int(hi - 1 - diff[-1]),
                B0=plan["levels"][0]["B"], B_last=plan["levels"][-1]["B"])


def _calls(sizes):
    return lambda ch, x: _run_calls(ch, x, sizes)


def _fir_len(poisons, taps, Bl, latency, F):
    return max(n for _, n in poisons) + taps + 2 * Bl + latency + 2 * F + 77


@pytest.mark.parametrize("case", list(FIR_CASES))
def test_fir_plan_paths_nonfinite(gpu_lib, case):
    """FIR_CASES on the flat family, per-channel taps, whole calls: multi-level (64, 300, 1000 frames), single level
    at 2048 / 4096 with batch depths 4, 6, 8, far tiers 8, 12, 16 (staggered, whole, two classes), merge, pipe, bulk;
    at least 8 channels, so that every position of _fir_poisons has a channel of its own.

    Fixed by this test (k_fir_mac_batch, k_fir_pipe's batch share, k_fir_mac_bulk): those kernels slide a window of T
    filter rows along the FDL rows and multiplied every row with every period's filter row, a zero spectrum where the
    row is outside that period's window.  0 x NaN = NaN, so a poisoned block reached every period of each launch that
    read its row: the NaN outlived fir_nan_window's end by 0.5 (T = 8) to 3.5 blocks (T = 4), 11 with the far tier in
    two classes, two last-level blocks on the multi-level plans with a tail (multi_300: frame 65535 against a bound of
    58942), and in the bulk form it reached earlier blocks of the same call (bulk_32768: a NaN at frame 77824 changed
    frame 65536).  The kernels now skip the products with rows outside the window."""
    frames, taps, C, hint, envs, check = FIR_CASES[case]
    C = max(C, 8)
    B0 = fir_b0(hint or frames)
    chans = [c for c in (1, 2, 3, 5, 6) if c < C - 1 or (C <= 4 and c < C)][:max(1, C - 1)]
    poisons = _fir_poisons([frames] * 8, B0, chans)
    Bl = 8192
    N = _fir_len(poisons, taps, Bl, 0, frames)
    N = -(-N // frames) * frames
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    h = ir_family("flat", taps, C)
    x = dyadic_signal(rng, N, C)
    sizes = [frames] * (N // frames)
    make = lambda: gpu_lib.Chain(48000, C).add_fir(h, block_hint=hint)
    want, got, plan = _twice(make, x, poisons, _calls(sizes), envs)
    plan = plan[0]
    assert check(plan), (case, plan)
    _fir_check("fir/" + case, _cat(want, C), _cat(got, C), poisons, taps, plan)


NF_EDGES = ["fused/B64_T64", "fused/B2048_T2049", "tail/B2048_P11", "far/P48", "depth/T8_P19", "pipe/B2048_P11",
            "multi/B256_T40961", "levels/B64_cap8192", "latency/B64_T17_lat17", "latency/B4096_T255_lat12293",
            "cluster/B2048_P3_sel2-9of10"]


@pytest.mark.parametrize("case", NF_EDGES)
def test_fir_plan_edges_nonfinite(gpu_lib, case):
    """One FIR_EDGES case per group (fused P = 1 and 2, tail, far tier at P = 48, depth 8, pipeline kernel,
    multi-level, eight levels, latency ring at B0 = 64 and 4096, and a selector whose unselected channels must pass the
    sample through at exactly frame n), taps shared by all channels on every other case and per channel otherwise,
    in the ragged calls of test_fir_plan_edges_exact (head kernel, general path, stash)."""
    e = FIR_EDGES[case]
    T, C, hint, sel, lat, want_plan = e["taps"], e["C"], e["hint"], e["sel"], e["latency"], e["plan"]
    n_sel = C if sel is None else sum(sel)
    B0, Bl = want_plan["levels"][0]["B"], want_plan["levels"][-1]["B"]
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    sizes = _ragged_sizes(rng, sum(e["lead"]) + 80 * B0 + T + 2 * Bl + lat, B0, e["lead"])
    chans = [c for c in range(C) if c % 4 in (1, 2)][:3] if sel is None else [0, 3, 5]
    poisons = _fir_poisons(sizes, B0, chans)
    assert max(n for _, n in poisons) + T + 2 * Bl + lat <= sum(sizes), (case, poisons)
    shared = NF_EDGES.index(case) % 2 == 0
    h = ir_family("flat", T, 1 if shared else n_sel, seed=T)
    x = dyadic_signal(rng, sum(sizes), C)
    make = lambda: gpu_lib.Chain(48000, C).add_fir(h[:, 0] if shared else h, selector=sel, latency=lat, block_hint=hint)
    want, got, plan = _twice(make, x, poisons, _calls(sizes), e["envs"])
    plan = plan[0]
    for k, v in want_plan.items():
        assert plan[k] == v, (case, k, plan[k], v)
    _fir_check("fir_edge/" + case, _cat(want, C), _cat(got, C), poisons, T, plan, lat, sel)


def test_fir_replan_replays_the_poisoned_first_call(gpu_lib):
    """No block hint: the NaN arrives in the first, 7-frame call, planned at B0 = 64; the kept input, NaN included, is
    replayed through the plans of the 150- and 300-frame calls after it.  The stream recovers by the final plan's
    bound, and reset() clears the replay buffer with everything else."""
    C, taps = 3, 20000
    poisons = [(1, 3)]
    N = 11 * 4096 + 77
    sizes = [7, 150, 300, 9000]
    sizes += [2000] * ((N - sum(sizes)) // 2000) + [(N - sum(sizes)) % 2000]
    h = ir_family("flat", taps, C, seed=1)
    x = dyadic_signal(np.random.default_rng(taps), N, C)
    make = lambda: gpu_lib.Chain(48000, C).add_fir(h)
    want, got, plan = _twice(make, x, poisons, _calls(sizes), fresh=False)
    plan = plan[0]
    assert plan["replans"] == 2 and plan["levels"][0]["B"] == 256, plan
    _fir_check("fir/replan", _cat(want, C), _cat(got, C), poisons, taps, plan)


# ------------------------------------------------------------------------------------------------------------
# Resample
# ------------------------------------------------------------------------------------------------------------
def _rs_poisons(sizes, C, in_len):
    """First frame of the fourth call, the middle of a multi-tile call, the last frame of a call, on the last channel
    (the part-filled channel tile), channel 1 and the middle one."""
    starts = np.concatenate([[0], np.cumsum(sizes)])
    big = max(range(len(sizes)), key=lambda j: sizes[j])
    pos = [int(starts[3]), int(starts[big]) + sizes[big] // 2, int(starts[5]) - 1]
    chans = sorted({C - 1, 1, C // 2} - {0}) if C > 2 else [C - 1]
    return [(k, pos[i % 3]) for i, k in enumerate(chans)]


def _rs_check(name, gpu_lib, fi, fo, bw, want, got, counts, poisons, tile):
    p = gpu_lib.resample_params(fi, fo, bw)
    Q = rs_expect_launch(want.shape[1], tile, 1, 1)["Q"]   # output frames per CTA of the tile that ran
    _isolated(want, got, poisons, name)
    for k, n in poisons:
        exact, near = rs_nan_windows(n, counts, p["n"], p["d"], p["in_len"], p["out_delay"], Q)
        diff = _differs(want[:, k], got[:, k])
        assert diff.any(), (name, k, n, "the sample never reached the output")
        bad = np.nonzero(diff & ~near)[0]
        assert bad.size == 0, (name, k, n, "outputs outside the tiles that read row n differ", bad[:8])
        assert np.all(np.isfinite(got[~near, k])), (name, k, n)
        idx, ex = np.nonzero(diff)[0], np.nonzero(exact)[0]
        _record("nonfinite", name, op="resample", k=k, n=n, tile=tile, before=int(max(ex[0] - idx[0], 0)) if ex.size else -1,
                after=int(max(idx[-1] - ex[-1], 0)) if ex.size else -1)


def _rs_run(sizes, poll=None):
    def run(ch, x):
        outs = _run_calls(ch, x, sizes)
        return outs + (_drain(ch, poll) if poll else [])
    return run


def _rs_case(gpu_lib, name, fi, fo, C, sizes, force=None, poll=None, bw=0.939, seed=0):
    base = rs_bases(fi, fo, bw, sum(sizes), seed=seed)
    x = _tiled(base, C)
    poisons = _rs_poisons(sizes, C, gpu_lib.resample_params(fi, fo, bw)["in_len"])
    want, got, plan = _twice(lambda: _rs_chain(gpu_lib, fi, fo, C, bw, force), x, poisons, _rs_run(sizes, poll), fresh=not poll)
    tile = plan[0]["tile"]
    assert tile == rs_expect_launch(C, force or 0, 1, 1)["tile"], (name, plan)
    counts = [o.shape[0] for o in want]
    _rs_check(name, gpu_lib, fi, fo, bw, _cat(want, C), _cat(got, C), counts, poisons, tile)
    return plan[0]


RS_NF_SHAPES = {"mma": [4, 36, 132, 260], "pair": [2, 66], "single": [1, 33, 129]}
assert all(set(v) <= set(RS_SHAPES[k]) for k, v in RS_NF_SHAPES.items())


@pytest.mark.parametrize("shape", list(RS_NF_SHAPES))
def test_resample_variants_nonfinite(gpu_lib, shape):
    """44100 -> 48000, every DSP_B200_RS_TILE variant the channel count can run, on channel counts at the tile edges
    (a part-filled last warp, column and 128-channel tile); calls of 1, 7, in_len - 1, in_len, in_len + 1 and 4096
    frames, then the drain."""
    fi, fo = 44100, 48000
    in_len = gpu_lib.resample_params(fi, fo)["in_len"]
    sizes = [1, 7, in_len - 1, in_len, in_len + 1, 4096, 1, 4096, 3 * in_len]
    for C in RS_NF_SHAPES[shape]:
        seen = set()
        for force in range(8):
            tile = rs_expect_launch(C, force, 1, 1)["tile"]
            if tile in seen:
                continue
            seen.add(tile)
            _rs_case(gpu_lib, "rs/variants/C%d/tile%d" % (C, tile), fi, fo, C, sizes, force, poll=1000, seed=C)


def test_resample_warps_nonfinite(gpu_lib):
    """The tensor-core kernels at 4, 2 and 1 warps per CTA (call sizes scaled by the SM count, as in
    test_resample_warps_per_cta) on 132 channels, tiles 4-7."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = [k * sms for k in (4, 16, 26, 36, 50, 64)] + [3]
    for force in (4, 5, 6, 7):
        _rs_case(gpu_lib, "rs/warps/tile%d" % force, 44100, 48000, 132, sizes, force, seed=force)


@pytest.mark.parametrize("rates", [(44100, 48000), (48000, 8000)], ids=lambda r: "%d-%d" % r)
@pytest.mark.parametrize("C", [5, 8])
def test_resample_ratios_and_drain_nonfinite(gpu_lib, rates, C):
    """44.1k -> 48k and 48k -> 8k on the FMA (5 channels) and tensor-core (8) kernels, ragged calls, a poisoned sample
    in the last in_len frames, so that the drain emits it, polled 7 frames at a time."""
    fi, fo = rates
    in_len = gpu_lib.resample_params(fi, fo)["in_len"]
    rng = np.random.default_rng(fi + fo + C)
    sizes = [1, 7, in_len - 1, in_len, in_len + 1, 2 * in_len + 5]
    while sum(sizes) < 6 * in_len:
        sizes.append(int(rng.integers(1, 4097)))
    sizes.append(in_len - 3)   # the last call: its frames leave the stream through the drain
    base = rs_bases(fi, fo, 0.939, sum(sizes), seed=C)
    x = _tiled(base, C)
    starts = np.cumsum([0] + sizes)
    poisons = _rs_poisons(sizes, C, in_len)[:2] + [(0, int(starts[-2]) + in_len // 2)]
    poll = 7 if fo > fi else 4096
    # after reset() the drain is dry (its counters survive, as in the reference): compared with the clean chain's
    want, got, plan = _twice(lambda: _rs_chain(gpu_lib, fi, fo, C, 0.939), x, poisons, _rs_run(sizes, poll), fresh=False)
    counts = [o.shape[0] for o in want]
    _rs_check("rs/ratio/%d-%d/C%d" % (fi, fo, C), gpu_lib, fi, fo, 0.939, _cat(want, C), _cat(got, C), counts,
              poisons, plan[0]["tile"])


# ------------------------------------------------------------------------------------------------------------
# Biquad
# ------------------------------------------------------------------------------------------------------------
def _bq_coefs(gpu_lib, stages, C, identity=False):
    fs = 192000
    names = BQ_CASCADE[:stages]
    c = np.zeros((stages, C, 5))
    for s, nm in enumerate(names):
        t, f, a0, a1, a2, a3 = BQ_SECTIONS[nm]
        sec = gpu_lib.biquad_design(t, f, a0, a1, a2, a3)
        for ch in range(C):
            c[s, ch] = [1, 0, 0, 0, 0] if identity and (s + ch) % 3 == 0 else sec
    return fs, c


def _bq_poisons(sizes, C):
    """Channel 0 (its pair partner 1 clean) 1000 frames into a call (the first half of a split tile), channel 2 on a call's first frame, the last channel
    (a half-empty last pair when C is odd) on a call's last frame; calls from the third on."""
    starts = np.cumsum([0] + list(sizes))
    pos = [int(starts[2]) + min(1000, sizes[2] // 2), int(starts[3]), int(starts[5]) - 1]
    chans = [0, 2, C - 1] if C >= 5 else [0, 2] if C >= 3 else [C - 1]
    return [(k, pos[i]) for i, k in enumerate(chans)]


def bq_case(gpu_lib, name, stages, C, sizes, identity=False, absorb=False):
    """The four properties on one biquad chain (also run in subprocesses under the process-wide knobs)."""
    from oracle import restate
    fs, coefs = _bq_coefs(gpu_lib, stages, C, identity)
    x = np.tile(np.random.default_rng(stages + C).standard_normal((sum(sizes), 1)) * 0.3, (1, C))
    x += np.arange(C)[None, :] * 1e-3
    poisons = _bq_poisons(sizes, C)

    def make():
        if not absorb:
            return gpu_lib.Chain(fs, C).add_biquad(coefs)
        a, b = gpu_lib.Chain(fs, C).add_biquad(coefs[:stages // 2]), gpu_lib.Chain(fs, C).add_biquad(coefs[stages // 2:])
        a.absorb(b)
        b.close()
        assert a.n_ops == 1
        return a
    want, got, plan = _twice(make, x, poisons, _calls(sizes))
    # the form of the last call, under the knobs the library read from this process's environment
    knob = lambda v: int(os.environ[v]) if v in os.environ else None
    form = bq_expect_launch(C, stages, sizes[-1], knob("DSP_B200_BQ_CH"), knob("DSP_B200_BQ_SPLIT"))
    assert (plan[0]["ch"], plan[0]["split"]) == (form["ch"], form["split"]), (name, plan)
    want, got = _cat(want, C), _cat(got, C)
    _isolated(want, got, poisons, name)
    ks = [k for k, _ in poisons]
    _, bad = _poisoned(x, poisons)
    ref = restate.biquad_cascade(bad[:, ks], coefs[:, ks])
    for j, (k, n) in enumerate(poisons):
        assert np.array_equal(got[:n, k], want[:n, k]), (name, k, n, "differs before n")
        m_gpu, m_ref = ~np.isfinite(got[n:, k]), ~np.isfinite(ref[n:, j])
        assert m_ref[0] and np.array_equal(m_gpu, m_ref), (name, k, n, int(np.sum(m_gpu)), int(np.sum(m_ref)))
        _record("nonfinite", name, op="biquad", k=k, n=n, nonfinite=int(np.sum(m_gpu)), frames=int(m_gpu.size))


BQ_NF = {
    "split_1st": (1, 4, [2048] * 6),
    "split_2st_ragged": (2, 5, [1000, 2048, 2047, 1, 2048, 1500, 2048]),
    "wide_2st": (2, 3, [4096] * 6),
    "wide_16st_257ch": (16, 257, [4095] * 5),
    "identity_5st": (5, 6, [4096, 2048, 4097, 3000, 4096, 4096]),
}


@pytest.mark.parametrize("case", list(BQ_NF))
def test_biquad_nonfinite(gpu_lib, case):
    """The default forms (split at calls of at most 2048 frames, 16-warp above) on 1, 2 and 16 stages, 257 channels
    (a half-empty last pair) and per-channel identity sections: the poisoned channel is non-finite from n to the end,
    as in the reference's recurrence, and nothing before n or on another channel moves."""
    stages, C, sizes = BQ_NF[case]
    bq_case(gpu_lib, "biquad/" + case, stages, C, sizes, identity=case.startswith("identity"))


def test_biquad_fused_pair_nonfinite(gpu_lib):
    """Two neighbouring cascades fused by absorb() into one 16-stage operator."""
    bq_case(gpu_lib, "biquad/absorb", 16, 4, [4096, 4096, 2048, 4096, 4096, 4096], absorb=True)


BQ_KNOBS = {
    "split_forced": (dict(DSP_B200_BQ_SPLIT="1"), 2, 4, [4096, 4096, 8192, 4096, 6000, 4096]),
    "ch1": (dict(DSP_B200_BQ_CH="1"), 2, 5, [4096, 2048, 4096, 4096, 4096, 4096]),
    "ch4": (dict(DSP_B200_BQ_CH="4"), 2, 9, [4096, 2048, 4096, 4096, 4096, 4096]),
}


@pytest.mark.parametrize("knob", list(BQ_KNOBS))
def test_biquad_forms_nonfinite_in_subprocess(knob):
    """DSP_B200_BQ_SPLIT=1 with calls above 2048 frames (the NaN of the first half reaches the second half's CTA through
    the published xstate / flag) and DSP_B200_BQ_CH=1 and 4: the library reads these once per process, so each case
    runs in a process of its own with the variable set."""
    envs, stages, C, sizes = BQ_KNOBS[knob]
    code = ("import sys; sys.path[:0] = [%r, %r]; import dsp_b200, test_gpu_nonfinite as t; dsp_b200.lib(); "
            "t.bq_case(dsp_b200, %r, %d, %d, %r)" % (ROOT, os.path.join(ROOT, "tests"), "biquad/" + knob, stages, C, sizes))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **envs), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]


# ------------------------------------------------------------------------------------------------------------
# Gain and align
# ------------------------------------------------------------------------------------------------------------
def _one_frame(name, want, got, poisons, at):
    _isolated(want, got, poisons, name)
    for k, n in poisons:
        diff = np.nonzero(_differs(want[:, k], got[:, k]))[0].tolist()
        t = at(k, n)
        assert diff == ([t] if 0 <= t < got.shape[0] else []), (name, k, n, diff[:8])
        assert np.sum(~np.isfinite(got[:, k])) == len(diff), (name, k, n)


def test_gain_nonfinite(gpu_lib):
    """y = mult x + add, mult = 0 on the poisoned channels 1 (0 x Inf = NaN, as in the reference) and 3: one
    non-finite frame, at n."""
    C = 6
    mult, add = [0.5, 0.0, -2.0, 0.0, 1.0, 3.0], [0.1, 0.0, 0.3, 0.2, 0.0, -1.0]
    sizes = [1, 4095, 4096, 4097, 100, 4096]
    x = np.random.default_rng(3).standard_normal((sum(sizes), C))
    poisons = [(1, 4096), (2, 8191), (3, 5000), (4, 0)]
    want, got, _ = _twice(lambda: gpu_lib.Chain(48000, C).add_gain(mult, add), x, poisons, _calls(sizes))
    _one_frame("gain", _cat(want, C), _cat(got, C), poisons, lambda k, n: n)


def test_align_nonfinite(gpu_lib):
    """Per-channel delays d_k and a discard of 1000 frames: the sample leaves at output frame n + d_k - 1000, and not at
    all when that is before the discard ends (channel 1: n + d_k < 1000)."""
    C = 5
    delays, discard = [0, 3, 700, 5000, 64], 1000
    sizes = [1, 999, 1, 4096, 3000, 4096, 4096, 4096]
    x = np.random.default_rng(4).standard_normal((sum(sizes), C))
    poisons = [(1, 500), (2, 5000), (3, 10), (4, 1000), (0, 1001)]
    want, got, _ = _twice(lambda: gpu_lib.Chain(48000, C).add_align(delays, discard), x, poisons, _calls(sizes))
    _one_frame("align", _cat(want, C), _cat(got, C), poisons, lambda k, n: n + delays[k] - discard)


# ------------------------------------------------------------------------------------------------------------
# One composed chain
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("slabs,mode", [(1, "host"), (1, "submit"), (1, "device"), (2, "host"), (3, "device")])
def test_composed_chain_nonfinite(gpu_lib, slabs, mode):
    """Chain A of test_gpu_chain (gain, 20 biquad stages, resample 44.1k -> 48k, per-channel FIR with a channel passed
    through, biquad, align) on 7 channels in 1, 2 and 3 slabs: a NaN on channel 1 (slab 0) and an Inf on channel 5 (the
    FIR's unselected channel) leave the other channels and slabs bit-identical, through the stream and the drain; after
    reset() the stream and a dry drain are a fresh chain's."""
    from test_gpu_chain import _add_ops, _drain_all, _inputs, _run_device, _run_host, _run_submit, _spec
    C = 7
    fs, ops = _spec(gpu_lib, "A", C)
    xs = _inputs("A", C)
    sizes = [x.shape[0] for x in xs]
    x = np.concatenate(xs)
    starts = np.cumsum([0] + sizes)
    poisons = [(1, int(starts[5]) + 1000), (5, int(starts[7]) + 3)]
    call = {"host": _run_host, "submit": lambda ch, v: _run_submit(gpu_lib, ch, v), "device": _run_device}[mode]

    clean, bad = _poisoned(x, poisons)

    def run(ch, xx):
        outs = call(ch, np.split(xx, starts[1:-1])) + _drain_all(ch)
        ch.reset()
        return outs + ["reset"] + _run_host(ch, np.split(clean, starts[1:-1])) + _drain_all(ch)

    def make():
        ch = _add_ops(gpu_lib.Chain(fs, C, slabs_per_device=slabs), ops)
        assert ch.n_shards == slabs
        return ch
    a, b = make(), make()
    try:
        want, got = run(a, clean), run(b, bad)
    finally:
        a.close()
        b.close()
    r = next(i for i, o in enumerate(want) if isinstance(o, str))
    assert isinstance(got[r], str)
    _same_calls(got[r + 1:], want[r + 1:], "the stream after reset()")
    # the stream after reset() is a fresh chain's clean stream (the drain after it stays dry: its counters survive)
    f = make()
    try:
        fresh = _run_host(f, np.split(clean, starts[1:-1]))
    finally:
        f.close()
    _same_calls(got[r + 1:r + 1 + len(xs)], fresh, "a fresh chain's stream")
    assert got[-1] is None and all(o is None for o in got[r + 1 + len(xs):]), "the drain after reset() is not dry"
    w, g = _cat(want[:r], C), _cat(got[:r], C)
    _isolated(w, g, poisons, "chain/%d/%s" % (slabs, mode))
    for k, _ in poisons:
        assert not np.all(np.isfinite(g[:, k])), k
