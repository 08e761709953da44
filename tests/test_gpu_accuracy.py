"""GPU tier: the kernels against extended-precision truths, with error bounds scaled to the signal.

FIR: dyadic signals and taps, so that the exact convolution is known (accuracy.exact_conv); three IR families
(flat random taps, an envelope that rises toward the last tap, a comb with distinct weights either side of every
multiple of 64 taps -- every partition boundary of every plan), through every plan the library makes.
Bound: normalized RMS <= 1e-14, normalized max <= 1e-13 (scale = rms(x) ||h||_2 per channel).  Measured on an
H100 80GB HBM3 (400 W limit), worst over every FIR case below: RMS 4.8e-16, max 3.3e-15.

Biquad: ill-conditioned sections (poles near z = 1: corners down to 5 Hz at up to 192 kHz) on large, slow
inputs, against an 80-bit long-double run of the same coefficients.  Bound per channel:
err_gpu <= max(4 err_ref64, 64 u rms(truth)), where err_ref64 is the error of the reference's own FP64
recurrence (restate.biquad_cascade) and u = 2^-53.

Errors of each case are appended as JSON lines to the file DSP_B200_ACCURACY_LOG names, when it is set.
"""
import json
import os
import zlib

import numpy as np
import pytest

from accuracy import H_MAX, biquad_within_ref, dyadic_signal, dyadic_taps, env, exact_conv, fir_nerr

pytestmark = pytest.mark.gpu
FIR_RMS, FIR_MAX = 1e-14, 1e-13


def _record(kind, name, **vals):
    """Measured errors, one JSON line per case, when DSP_B200_ACCURACY_LOG names a file."""
    path = os.environ.get("DSP_B200_ACCURACY_LOG")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps(dict(kind=kind, name=name, **vals)) + "\n")


# ------------------------------------------------------------------------------------------------------------
# FIR
# ------------------------------------------------------------------------------------------------------------
H_SHIFT = 12


def ir_family(family, taps, channels, seed=0):
    """[taps, channels] dyadic taps (h = j 2^-12, |j| <= 2^12), distinct per channel."""
    rng = np.random.default_rng(1000 + seed)
    n = np.arange(taps)[:, None]
    if family == "flat":
        h = rng.uniform(-1, 1, (taps, channels))
    elif family == "rising":
        h = rng.uniform(-1, 1, (taps, channels)) * np.exp(6.9 * (n - taps + 1) / taps)
    else:
        # comb: taps 64 q - 1, 64 q, 64 q + 1 for every q, and the very last tap, all with distinct weights
        pos = sorted({p for q in range(taps // 64 + 1) for p in (64 * q - 1, 64 * q, 64 * q + 1) if 0 <= p < taps} | {taps - 1})
        h = np.zeros((taps, channels))
        vals = np.concatenate([np.arange(-H_MAX, 0), np.arange(1, H_MAX + 1)])
        for c in range(channels):
            h[pos, c] = rng.permutation(vals)[:len(pos)]
    return dyadic_taps(h, H_SHIFT)



# name: (call frames, taps, channels, block_hint, env, plan check)
F4, F2 = 4096, 2048


def _single(B, P=None):
    return lambda p: len(p["levels"]) == 1 and p["levels"][0]["B"] == B and (P is None or p["levels"][0]["P"] == P)


FIR_CASES = {
    "multi_64": (64, 20000, 4, 0, {}, lambda p: len(p["levels"]) > 1 and p["levels"][0]["B"] == 64),
    "multi_300": (300, 50000, 4, 0, {}, lambda p: len(p["levels"]) > 1 and p["levels"][0]["B"] == 256),
    "multi_1000": (1000, 131072, 4, 0, {}, lambda p: len(p["levels"]) > 1 and p["levels"][0]["B"] == 512),
    "single_2048_t4": (F2, 131072, 8, F2, dict(DSP_B200_FIR_T=4), lambda p: _single(F2, 64)(p) and p["t_batch"] == 4),
    "single_2048_t6": (F2, 131072, 8, F2, dict(DSP_B200_FIR_T=6), lambda p: _single(F2, 64)(p) and p["t_batch"] == 6),
    "single_2048_t8": (F2, 131072, 8, F2, dict(DSP_B200_FIR_T=8), lambda p: _single(F2, 64)(p) and p["t_batch"] == 8),
    "single_4096_t4": (F4, 131072, 8, F4, dict(DSP_B200_FIR_T=4), lambda p: _single(F4, 32)(p) and p["t_batch"] == 4),
    "single_4096_t6": (F4, 131072, 8, F4, dict(DSP_B200_FIR_T=6), lambda p: _single(F4, 32)(p) and p["t_batch"] == 6),
    "single_4096_t8": (F4, 131072, 8, F4, dict(DSP_B200_FIR_T=8), lambda p: _single(F4, 32)(p) and p["t_batch"] == 8),
    "merge": (F4, 131072, 8, F4, dict(DSP_B200_FIR_MERGE=1), lambda p: _single(F4, 32)(p) and p["merge"] == 1),
    "pipe_4096": (F4, 131072, 8, F4, dict(DSP_B200_FIR_PIPE=1), lambda p: _single(F4, 32)(p) and p["pipe"] == 1),
    "pipe_2048": (F2, 70000, 8, F2, dict(DSP_B200_FIR_PIPE=1), lambda p: _single(F2)(p) and p["pipe"] == 1),
    "bulk_32768": (32768, 50000, 3, 32768, {}, lambda p: p["levels"] == [{"B": 8192, "P": 7}]),
}
for _far in (8, 12, 16):
    for _mode, _e in (("s", dict(DSP_B200_FIR_STAGGER=1)), ("u", dict(DSP_B200_FIR_STAGGER=0)),
                      ("u2", dict(DSP_B200_FIR_STAGGER=0, DSP_B200_FIR_FAR_CLASSES=2))):
        if _mode == "u2" and (_far // 2) % 4:
            continue   # two classes need t_far / 2 to be a multiple of t_batch (4): far tiers 8 and 16
        _e = dict(_e, DSP_B200_FIR_T2=_far, DSP_B200_FIR_T=4)
        _cls = 2 if _mode == "u2" else 1
        FIR_CASES["far%d_%s" % (_far, _mode)] = (
            F2, 131072, 8, F2, _e,
            (lambda far, stag, cls: lambda p: _single(F2, 64)(p) and p["t_far"] == far and p["stagger"] == stag
             and (stag or p["far_classes"] == cls))(_far, 1 if _mode == "s" else 0, _cls))


def _run_fir(gpu_lib, x, h, frames, hint, envs, selector=None, latency=0, cuts=None):
    C = x.shape[1]
    with env(**envs):
        ch = gpu_lib.Chain(48000, C).add_fir(h if h.shape[1] > 1 else h[:, 0], selector=selector, latency=latency, block_hint=hint)
        if cuts is None:
            cuts = list(range(0, x.shape[0], frames)) + [x.shape[0]]
        got = np.concatenate([ch.run(x[a:b]).copy() for a, b in zip(cuts[:-1], cuts[1:])])
        plan = ch.describe()[0]
    return ch, got, plan


@pytest.mark.parametrize("family", ["flat", "rising", "comb"])
@pytest.mark.parametrize("case", list(FIR_CASES))
def test_fir_plan_paths_exact(gpu_lib, case, family):
    """Every plan path against the exact convolution: multi-level plans (64-, 300- and 1000-frame calls), a single
    level at 2048 and 4096 frames with batch depths 4, 6 and 8, far tiers 8, 12 and 16 (staggered, whole launches,
    two classes), the merged MAC grid, the pipeline kernel, and the bulk form.  Measured (H100 80GB HBM3, 400 W), worst
    over cases and families: normalized RMS 4.8e-16, max 3.3e-15."""
    frames, taps, C, hint, envs, check = FIR_CASES[case]
    rng = np.random.default_rng(zlib.crc32((case + family).encode()))
    N = max(48 * 4096 if taps >= 100000 else taps + 8 * max(frames, 4096), 3 * frames) + 77
    h = ir_family(family, taps, C)
    x = dyadic_signal(rng, N, C)
    want = exact_conv(x, h, H_SHIFT)
    ch, got, plan = _run_fir(gpu_lib, x, h, frames, hint, envs)
    ch.close()
    assert check(plan), (case, plan)
    r, m = fir_nerr(got, want, x, h)
    _record("fir", "%s/%s" % (case, family), rms=r, max=m)
    assert r <= FIR_RMS and m <= FIR_MAX, (case, family, r, m, plan)


@pytest.mark.parametrize("family", ["flat", "comb"])
@pytest.mark.parametrize("case", ["cluster", "window", "scattered", "latency", "ragged_reset", "pipe_300"])
def test_fir_block_io_and_stream_shapes_exact(gpu_lib, case, family):
    """Direct block I/O (clusters of four contiguous channels, a window of channels, a scattered selector),
    fir's latency ring, ragged calls mixed with whole blocks with one reset() mid-stream, and the pipeline kernel
    on 300 channels (CTAs that walk two or three channels; channels either side of 132 and 264 sampled).  Measured
    (H100 80GB HBM3, 400 W): within the worst figures of test_fir_plan_paths_exact."""
    F, taps = 4096, 40000
    rng = np.random.default_rng(zlib.crc32((case + family).encode()))
    C = {"cluster": 8, "window": 12, "scattered": 12, "latency": 8, "ragged_reset": 5, "pipe_300": 300}[case]
    sel = None
    if case == "window":
        sel = [4 <= c < 12 for c in range(C)]
    if case == "scattered":
        sel = [c in (1, 2, 3, 5, 6, 7, 10, 11) for c in range(C)]
    n_sel = C if sel is None else sum(sel)
    lat = 24576 if case == "latency" else 0
    envs = dict(DSP_B200_FIR_PIPE=1) if case == "pipe_300" else {}
    N = 20 * F + 100
    if case == "pipe_300":
        taps, N = 30000, 17 * F
        h = np.tile(ir_family(family, taps, 5), (1, (C + 4) // 5))[:, :C]
    else:
        h = ir_family(family, taps, n_sel)
    x = dyadic_signal(rng, N, C)
    cuts = None
    if case == "ragged_reset":
        cuts = sorted(set([0, N, 3 * F, 4 * F, 5 * F, 9 * F, 10 * F] + list(rng.integers(1, N, 12))))
    ch, got, plan = _run_fir(gpu_lib, x, h, F, F, envs, selector=sel, latency=lat, cuts=cuts)
    assert len(plan["levels"]) == 1 and plan["pipe"] == (1 if case == "pipe_300" else 0), plan
    worst = []
    if case == "pipe_300":
        cs = [0, 1, 131, 132, 133, 263, 264, 265, 299]
        want = exact_conv(x[:, cs], h[:, cs], H_SHIFT)
        worst.append(fir_nerr(got[:, cs], want, x[:, cs], h[:, cs]))
    else:
        want = exact_conv(x, h, H_SHIFT, selector=sel, latency=lat)
        worst.append(fir_nerr(got, want, x, h, selector=sel))
        if sel is not None:
            for c in range(C):
                if not sel[c]:
                    assert np.array_equal(got[:, c], x[:, c])
        if case == "ragged_reset":
            # reset mid-stream: the stream starts again from silence, in whole blocks and ragged calls
            ch.reset()
            cuts2 = [0, F, F + 1, 2 * F, 3 * F - 5, 6 * F, 8 * F]
            got2 = np.concatenate([ch.run(x[a:b]).copy() for a, b in zip(cuts2[:-1], cuts2[1:])])
            worst.append(fir_nerr(got2, want[:8 * F], x[:8 * F], h))
    ch.close()
    r, m = max(w[0] for w in worst), max(w[1] for w in worst)
    _record("fir", "%s/%s" % (case, family), rms=r, max=m)
    assert r <= FIR_RMS and m <= FIR_MAX, (case, family, r, m, plan)


# ------------------------------------------------------------------------------------------------------------
# Biquad
# ------------------------------------------------------------------------------------------------------------
# (type, fs, arg0, arg1, arg2, arg3): biquad_design's arguments (types as in include/dsp_b200.h)
BQ_SECTIONS = {
    "lowpass_80_48k": (7, 48000, 80.0, 0.707, 0.0, 0.0),
    "lowpass_20_96k_q0.5": (7, 96000, 20.0, 0.5, 0.0, 0.0),
    "lowpass_40_192k": (7, 192000, 40.0, 0.707, 0.0, 0.0),
    "lowpass_10_192k": (7, 192000, 10.0, 0.707, 0.0, 0.0),
    "lowpass_10_192k_q5": (7, 192000, 10.0, 5.0, 0.0, 0.0),
    "highpass_5_44k_q0.5": (8, 44100, 5.0, 0.5, 0.0, 0.0),
    "highpass_10_192k_q10": (8, 192000, 10.0, 10.0, 0.0, 0.0),
    "lowpass1_10_96k": (1, 96000, 10.0, 0.707, 0.0, 0.0),
    "highpass1_5_192k": (2, 192000, 5.0, 0.707, 0.0, 0.0),
    "allpass1_10_48k": (3, 48000, 10.0, 0.707, 0.0, 0.0),
    "lowshelf1_10_192k_+15": (4, 192000, 10.0, 0.707, 15.0, 0.0),
    "highshelf1_20_96k_-15": (5, 96000, 20.0, 0.707, -15.0, 0.0),
    "bandpass_skirt_10_192k_q2": (9, 192000, 10.0, 2.0, 0.0, 0.0),
    "bandpass_peak_20_96k_q0.5": (10, 96000, 20.0, 0.5, 0.0, 0.0),
    "notch_10_192k_q10": (11, 192000, 10.0, 10.0, 0.0, 0.0),
    "allpass_10_192k": (12, 192000, 10.0, 0.707, 0.0, 0.0),
    "peak_8_192k_q0.5_+15": (13, 192000, 8.0, 0.5, 15.0, 0.0),
    "peak_30_44k_q10_-15": (13, 44100, 30.0, 10.0, -15.0, 0.0),
    "lowshelf_10_96k_-15": (14, 96000, 10.0, 0.707, -15.0, 0.0),
    "highshelf_20_192k_+12": (15, 192000, 20.0, 1.0, 12.0, 0.0),
    "linkwitz_30_to_10_192k": (16, 192000, 30.0, 0.707, 10.0, 0.5),
}


def bq_inputs(fs, frames, seed=0):
    """[frames, 4]: low sines near full scale, a DC step 0 -> 0.9, the reference sweep, noise."""
    from oracle import restate
    rng = np.random.default_rng(seed)
    t = np.arange(frames) / fs
    x = np.zeros((frames, 4))
    x[:, 0] = 0.45 * np.sin(2 * np.pi * 7.0 * t) + 0.4 * np.sin(2 * np.pi * 31.0 * t + 1.0) + 0.05 * np.sin(2 * np.pi * 440.0 * t)
    x[frames // 7:, 1] = 0.9
    x[:, 2] = restate.sgen_sine(fs, 1, frames, 5.0, 20000.0)[:, 0] * 0.9
    x[:, 3] = rng.standard_normal(frames) * 0.3
    return x


def bq_check(name, got, x, coefs):
    """Per channel: err_gpu <= max(4 err_ref64, 64 u rms(truth)) (accuracy.biquad_within_ref)."""
    for c, (e_gpu, e_ref, ratio) in enumerate(biquad_within_ref(got, x, coefs)):
        _record("biquad", "%s/ch%d" % (name, c), err_gpu=e_gpu, err_ref64=e_ref, ratio=ratio)


def _design(gpu_lib, sec):
    t, fs, a0, a1, a2, a3 = sec
    return gpu_lib.biquad_design(t, fs, a0, a1, a2, a3)


@pytest.mark.parametrize("form", ["split", "wide"])
@pytest.mark.parametrize("name", list(BQ_SECTIONS))
def test_biquad_ill_conditioned_sections(gpu_lib, name, form):
    """One section, four slow, large inputs; calls of 2048 frames (split form) or 4096 (16-warp form), ragged calls
    after a reset.  Measured (H100 80GB HBM3, 400 W): err_gpu at most 0.25 of its bound in every case.  The 10 Hz /
    192 kHz lowpass with Q 5 is at most 2.9e-12 relative over its inputs (the FP64 recurrence: up to 1.6e-10); with
    the scan in the companion basis (before biquad.cu's basis change) it was 1.4e-9 on the sine input."""
    sec = BQ_SECTIONS[name]
    fs = sec[1]
    coefs = _design(gpu_lib, sec)[None, :]
    N = 6 * 4096 + 1
    x = bq_inputs(fs, N, seed=len(name))
    F = 2048 if form == "split" else 4096
    ch = gpu_lib.Chain(fs, 4).add_biquad(coefs)
    got = np.concatenate([ch.run(x[i:i + F]).copy() for i in range(0, N, F)])
    bq_check("%s/%s" % (name, form), got, x, coefs)
    ch.reset()
    cuts = [0, 1, 2047, 2049, 4096, 8192, 8193, 12287, 16384, N] if form == "split" else [0, 4095, 8191, 8192, 12289, 20000, N]
    got2 = np.concatenate([ch.run(x[a:b]).copy() for a, b in zip(cuts[:-1], cuts[1:])])
    bq_check("%s/%s/ragged" % (name, form), got2, x, coefs)
    ch.close()


BQ_CASCADE = ["lowpass_10_192k_q5", "highpass_10_192k_q10", "lowshelf1_10_192k_+15", "notch_10_192k_q10",
              "peak_8_192k_q0.5_+15", "lowpass_10_192k", "allpass_10_192k", "bandpass_skirt_10_192k_q2",
              "highshelf_20_192k_+12", "linkwitz_30_to_10_192k", "lowpass_40_192k", "highpass1_5_192k",
              "lowpass1_10_96k", "allpass1_10_48k", "highshelf1_20_96k_-15", "lowpass_20_96k_q0.5"]


@pytest.mark.parametrize("stages,channels,call", [(1, 1, 4096), (2, 3, 8192), (16, 3, 4097), (16, 257, 4095), (2, 257, 2048), (16, 1, 8191)])
def test_biquad_cascades_channels_and_tiles(gpu_lib, stages, channels, call):
    """1, 2 and 16 ill-conditioned stages (192 kHz), 1, 3 and 257 channels (a half-empty last CTA), calls at tile
    boundaries (4096, 8192, +-1 frame), then reset() and the same stream again in ragged calls.  Measured (H100 80GB
    HBM3, 400 W): worst 1.0e-11 relative (16 stages), against 8.3e-11 for the FP64 recurrence."""
    fs = 192000
    coefs = np.array([_design(gpu_lib, BQ_SECTIONS[n]) for n in BQ_CASCADE[:stages]])
    N = 3 * 8192 + 5
    base = bq_inputs(fs, N, seed=stages)
    x = np.tile(base, (1, (channels + 3) // 4))[:, :channels]
    ch = gpu_lib.Chain(fs, channels).add_biquad(coefs)
    got = np.concatenate([ch.run(x[i:i + call]).copy() for i in range(0, N, call)])
    ch.reset()
    cuts = [0, 100, 4096, 4097, 8192, 8191 + 4096, 2 * 8192, N]
    got2 = np.concatenate([ch.run(x[a:b]).copy() for a, b in zip(cuts[:-1], cuts[1:])])
    ch.close()
    # channels that carry the same signal agree bit for bit whichever CTA computed them
    for c in range(4, channels):
        assert np.array_equal(got[:, c], got[:, c % 4])
    k = min(channels, 4)
    bq_check("cascade%d_ch%d_call%d" % (stages, channels, call), got[:, :k], base[:, :k], coefs)
    bq_check("cascade%d_ch%d_ragged" % (stages, channels), got2[:, :k], base[:, :k], coefs)


def test_biquad_per_channel_identity_sections_and_fused_neighbours(gpu_lib):
    """Per-channel coefficients with identity sections {1, 0, 0, 0, 0} where a stage does not act on a channel, and
    two neighbouring cascades (a chain absorbing the next one) fused into one operator."""
    fs, C = 192000, 4
    names = ["lowpass_10_192k_q5", "notch_10_192k_q10", "peak_8_192k_q0.5_+15", "highpass_10_192k_q10", "allpass_10_192k"]
    coefs = np.zeros((len(names), C, 5))
    for s, n in enumerate(names):
        for c in range(C):
            coefs[s, c] = _design(gpu_lib, BQ_SECTIONS[n]) if (s + c) % 3 else [1, 0, 0, 0, 0]
    N = 5 * 4096 + 3
    x = bq_inputs(fs, N, seed=9)
    ch = gpu_lib.Chain(fs, C).add_biquad(coefs[:2])
    nxt = gpu_lib.Chain(fs, C).add_biquad(coefs[2:])
    ch.absorb(nxt)           # neighbouring cascades of two chains become one operator
    assert ch.n_ops == 1
    got = np.concatenate([ch.run(x[i:i + 4096]).copy() for i in range(0, N, 4096)])
    ch.close()
    nxt.close()
    bq_check("per_channel_fused", got, x, coefs)
