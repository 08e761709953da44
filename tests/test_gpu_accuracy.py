"""GPU tier: the kernels against extended-precision truths, with error bounds scaled to the signal.

FIR: dyadic signals and taps, so that the exact convolution is known (accuracy.exact_conv); three IR families
(flat random taps, an envelope that rises toward the last tap, a comb with distinct weights either side of every
multiple of 64 taps -- every partition boundary of every plan), through every plan the library makes.
Bound: normalized RMS <= 1e-14, normalized max <= 1e-13 (scale = rms(x) ||h||_2 per channel).  Measured on an
H100 80GB HBM3 (400 W limit), worst over every FIR case below: RMS 4.8e-16, max 3.3e-15.

FIR plan edges (test_fir_plan_edges_exact and the two tests after it): every boundary fir_schedule() (fir_plan.h) draws,
each case asserting its plan and which paths ran, in whole blocks and then ragged calls after reset().  Measured on an H100
80GB HBM3 (700 W limit), worst normalized RMS / max per group: fused kernel without tail (P = 1, 2) 4.7e-16 /
2.7e-15; tail, batch and stagger thresholds 4.6e-16 / 2.7e-15; far tier at P = 47 / 48 4.7e-16 / 2.7e-15; batch
depths 6 and 8 4.2e-16 / 2.7e-15; pipeline kernel with and without batch 4.6e-16 / 2.5e-15; multi-level 4.3e-16 /
3.0e-15; eight levels 4.4e-16 / 2.8e-15; bulk 4.9e-16 / 2.9e-15; FFT tiles at CPB +- 1 4.5e-16 / 2.3e-15; cluster
fall-backs (selectors, misaligned device buffers) 4.7e-16 / 2.9e-15; latency ring 4.5e-16 / 2.6e-15; re-planning
4.2e-16 / 2.4e-15.

Biquad: ill-conditioned sections (poles near z = 1: corners down to 5 Hz at up to 192 kHz) on large, slow
inputs, against an 80-bit long-double run of the same coefficients.  Bound per channel:
err_gpu <= max(4 err_ref64, 64 u rms(truth)), where err_ref64 is the error of the reference's own FP64
recurrence (restate.biquad_cascade) and u = 2^-53.

Resample: the polyphase form against the long-double tap table and stream of accuracy.resample_truth, bound
normalized RMS <= 1e-14 and max <= 1e-13 (scale = rms(x) ||G|| per channel), scaled up for very long tables
(_table_factor).  Measured (H100 80GB HBM3, 400 W), worst per group: tap-table readback max 4.8e-15 ||G||; every
DSP_B200_RS_TILE variant at tile edges 1.4e-15 / 7.5e-15; warps per CTA 1.4e-15 / 7.1e-15; the 15 ratios at
bandwidth 0.7 2.8e-15 / 9.1e-15, at 0.99 1.0e-14 / 4.6e-14, at 0.999 1.5e-14 / 5.9e-14; stream shapes 6.0e-15 /
2.6e-14 (6:1).  Tiles 1-3 agree bit for bit with each other, and so do tiles 4-7.

Errors of each case are appended as JSON lines to the file DSP_B200_ACCURACY_LOG names, when it is set.
"""
import json
import os
import zlib

import numpy as np
import pytest

from accuracy import (F2, F4, FIR_CASES, FIR_EDGES, H_MAX, RS_RATIOS, RsPacing, _fir_plan, _ladder, biquad_within_ref, bq_expect_launch,
                      dyadic_signal, dyadic_taps, env, exact_conv, fir_nerr, resample_taps_truth, resample_truth, rs_counts, rs_expect_launch, rs_nerr,
                      taps_norm)

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


PATHS = ("fused", "cluster", "pipe", "bulk", "general")   # describe()["paths"]: level-0 blocks per path ("head": launches)


def _ragged_sizes(rng, N, B, lead=()):
    """Call sizes summing to N: `lead`, then from an aligned start B - 1, B, B + 1; B - 3 and six 1-frame calls across
    a block boundary; B - 6 and B + 6 (from offset B - 3 across two boundaries); then seeded sizes.  While the
    stream is young enough to be replayed (16384 frames) every call stays below 2 B, which would re-plan."""
    sizes = list(lead)
    pos = sum(sizes)
    if pos % B:
        sizes.append(B - pos % B)
    sizes += [B - 1, B, B + 1, B - 3] + [1] * 6 + [B - 6, B + 6]
    pos = sum(sizes)
    while pos < N:
        top = 2 * B - 1 if pos < 16384 + 2 * B else 4 * B + 7
        f = min(int(rng.integers(1, top + 1)), N - pos)
        sizes.append(f)
        pos += f
    return sizes


def _run_sizes(ch, x, sizes):
    return np.concatenate([o.copy() for o in _run_calls(ch, x, sizes)])


def _check_plan(p, want, case):
    for k, v in want.items():
        assert p[k] == v, (case, k, p[k], v, p)


def _edge_mixes(case):
    return ["flat-shared", "comb-channel"] + (["rising-shared"] if FIR_EDGES[case]["rising"] else [])


@pytest.mark.parametrize("case,mix", [(c, m) for c in FIR_EDGES for m in _edge_mixes(c)])
def test_fir_plan_edges_exact(gpu_lib, case, mix):
    """Every boundary of fir_schedule() against the exact convolution, with the plan each case must make asserted
    (describe()), in two passes of one chain: whole aligned blocks, then reset() and ragged calls (_ragged_sizes).
    describe()["paths"] must show which path each pass took.  Streams of at least 2 R + 3 blocks of the last level
    (R: FDL rows), so that every FDL and V-slot ring wraps; the `short` cases stop before the filter's length.  Taps
    flat and shared by all channels, comb and per channel, and rising and shared on threshold cases.  Measured
    (H100 80GB HBM3, 700 W): see the module docstring."""
    e = FIR_EDGES[case]
    family, taps_mode = mix.split("-")
    T, C, hint, sel, lat, want_plan = e["taps"], e["C"], e["hint"], e["sel"], e["latency"], e["plan"]
    n_sel = C if sel is None else sum(sel)
    B0 = want_plan["levels"][0]["B"]
    Bl, Pl = want_plan["levels"][-1]["B"], want_plan["levels"][-1]["P"]
    R = Pl + want_plan["bulk"] - 1
    N = max((2 * R + 3) * Bl, 16 * B0, 8 * lat + 4 * B0, sum(e["lead"]) + 8 * B0) + 77
    if e["short"]:
        N = T - 3 * B0 - 5
    rng = np.random.default_rng(zlib.crc32((case + mix).encode()))
    h = ir_family(family, T, 1 if taps_mode == "shared" else n_sel, seed=T)
    x = dyadic_signal(rng, N, C)
    want = exact_conv(x, h, H_SHIFT, selector=sel, latency=lat)
    with env(**e["envs"]):
        ch = gpu_lib.Chain(48000, C).add_fir(h if h.shape[1] > 1 else h[:, 0], selector=sel, latency=lat, block_hint=hint)
        call = e["call"] or B0
        NA = N // call * call
        got_a = _run_sizes(ch, x[:NA], [call] * (NA // call))
        pa = ch.describe()[0]
        ch.reset()
        got_b = _run_sizes(ch, x, _ragged_sizes(rng, N, B0, e["lead"]))
        pb = ch.describe()[0]
    ch.close()
    _check_plan(pa, want_plan, case)
    _check_plan(pb, want_plan, case)
    # whole aligned blocks: one path for all of them
    # (the cluster form: B0 >= 2048, an even channel count, selected channels contiguous -- as every selector here is --
    # in fours from an even one)
    cluster = B0 >= 2048 and C % 2 == 0 and n_sel % 4 == 0 and (sel is None or sel.index(True) % 2 == 0)
    path =("pipe" if want_plan["pipe"] else "bulk" if want_plan["bulk"] > 1 else
            ("cluster" if cluster else "fused") if want_plan["levels"][0]["P"] <= 2 or want_plan["tail_pf"] == 2 else "general")
    assert pa["paths"] == dict({k: 0 for k in PATHS + ("head",)}, **{path: NA // B0}), (case, path, pa["paths"])
    # ragged calls: the head kernel and the general path, every block by exactly one path
    d = {k: pb["paths"][k] - pa["paths"][k] for k in PATHS + ("head",)}
    assert d["head"] > 0 and d["general"] > 0 and sum(d[k] for k in PATHS) == N // B0, (case, d)
    if want_plan["bulk"] > 1:
        assert d["bulk"] > 0, (case, d)
    if sel is not None:
        for c in range(C):
            if not sel[c]:
                assert np.array_equal(got_a[:, c], x[:NA, c]) and np.array_equal(got_b[:, c], x[:, c]), (case, c)
    ra, ma = fir_nerr(got_a, want[:NA], x[:NA], h, selector=sel)
    rb, mb = fir_nerr(got_b, want, x, h, selector=sel)
    r, m = max(ra, rb), max(ma, mb)
    _record("fir", "edges/%s/%s" % (case, mix), group=case.split("/")[0], rms=r, max=m)
    assert r <= FIR_RMS and m <= FIR_MAX, (case, mix, ra, ma, rb, mb, pb)


@pytest.mark.parametrize("B,P", [(F2, 2), (F2, 3), (F4, 2), (F4, 3)])
def test_fir_cluster_form_falls_back_on_misaligned_device_buffers(gpu_lib, B, P):
    """run_device on torch buffers: whole blocks on 16-byte aligned rows take the cluster form; one whole block and
    two ragged calls on buffers offset by one double (8-byte aligned) take the per-channel form, the stash and the head
    kernel, which touch the caller's rows with 8-byte accesses only; the stream stays exact."""
    import torch
    C, T = 8, (P - 1) * B + 1
    rng = np.random.default_rng(B + P)
    h = ir_family("comb", T, C, seed=P)
    nblk = 2 * P + 6
    N = nblk * B
    x = dyadic_signal(rng, N, C)
    want = exact_conv(x, h, H_SHIFT)
    ch = gpu_lib.Chain(48000, C).add_fir(h, block_hint=B)
    st = torch.cuda.current_stream().cuda_stream
    d_x = torch.from_numpy(x.reshape(-1)).cuda()
    d_y = torch.zeros_like(d_x)
    odd_x = torch.zeros(2 * B * C + 1, dtype=torch.float64, device="cuda")
    odd_y = torch.zeros_like(odd_x)
    # (frames, misaligned) per call: aligned blocks, one misaligned block, aligned, two misaligned ragged calls, aligned
    calls = [(B, False)] * 3 + [(B, True)] + [(B, False)] * 2 + [(B // 2 - 3, True), (B // 2 + 3, True)]
    calls += [(B, False)] * (nblk - 7)
    pos = 0
    for f, odd in calls:
        a, b = pos * C, (pos + f) * C
        if odd:
            odd_x[1:1 + b - a] = d_x[a:b]
            assert (odd_x.data_ptr() + 8) % 16 == 8
            n = ch.run_device(0, f, odd_x.data_ptr() + 8, odd_y.data_ptr() + 8, st)
            d_y[a:b] = odd_y[1:1 + b - a]
        else:
            assert (d_x.data_ptr() + 8 * a) % 16 == 0
            n = ch.run_device(0, f, d_x.data_ptr() + 8 * a, d_y.data_ptr() + 8 * a, st)
        assert n == f
        pos += f
    torch.cuda.synchronize()
    got = d_y.cpu().numpy().reshape(N, C)
    p = ch.describe()[0]
    ch.close()
    _check_plan(p, _fir_plan([(B, P)], tail_pf=2 if P == 3 else 0), "misaligned")
    assert p["paths"] == dict(fused=1, cluster=nblk - 2, pipe=0, bulk=0, general=1, head=2), p["paths"]
    r, m = fir_nerr(got, want, x, h)
    _record("fir", "edges/misaligned/B%d_P%d" % (B, P), group="cluster", rms=r, max=m)
    assert r <= FIR_RMS and m <= FIR_MAX, (B, P, r, m)


@pytest.mark.parametrize("taps", [65, 20000])
def test_fir_replans_twice_then_keeps_its_plan(gpu_lib, taps):
    """No block hint: calls of 7, 150 and 300 frames plan B0 = 64, then re-plan to 128 and 256 (the kept input is
    replayed through each new plan); after the second re-plan the plan stays, through a 9000-frame call and through
    reset() with whole blocks and then ragged calls of up to 5000 frames."""
    C = 3
    steps = [(7, 64, 0), (150, 128, 1), (300, 256, 2), (9000, 256, 2)]
    plans = {65: {64: [(64, 2)], 128: [(128, 1)], 256: [(256, 1)]},
             20000: {B: _ladder(B, 4) for B in (64, 128, 256)}}[taps]
    rng = np.random.default_rng(taps)
    h = ir_family("flat", taps, C, seed=1)
    N = max(11 * 4096, 16 * 256) + 77
    x = dyadic_signal(rng, N, C)
    want = exact_conv(x, h, H_SHIFT)
    ch = gpu_lib.Chain(48000, C).add_fir(h)
    outs, pos = [], 0
    for f, B0, replans in steps:
        outs.append(ch.run(x[pos:pos + f]).copy())
        pos += f
        p = ch.describe()[0]
        assert [(L["B"], L["P"]) for L in p["levels"]] == plans[B0] and p["replans"] == replans, (f, p)
        assert p["tail_pf"] == (1 if taps == 20000 else 0), p
    sizes = []
    while pos + sum(sizes) < N:
        sizes.append(min(int(rng.integers(1, 2000)), N - pos - sum(sizes)))
    got = np.concatenate(outs + [_run_sizes(ch, x[pos:], sizes)])
    worst = [fir_nerr(got, want, x, h)]
    ch.reset()
    NA = N // 256 * 256
    worst.append(fir_nerr(_run_sizes(ch, x[:NA], [256] * (NA // 256)), want[:NA], x[:NA], h))
    ch.reset()
    worst.append(fir_nerr(_run_sizes(ch, x, _ragged_sizes(rng, N, 256, lead=(600, 1, 5000))), want, x, h))
    p = ch.describe()[0]
    ch.close()
    assert [(L["B"], L["P"]) for L in p["levels"]] == plans[256] and p["replans"] == 2, p
    r, m = max(w[0] for w in worst), max(w[1] for w in worst)
    _record("fir", "edges/replan/T%d" % taps, group="replan", rms=r, max=m)
    assert r <= FIR_RMS and m <= FIR_MAX, (taps, worst)


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
    after a reset.  describe() shows that every call of F frames ran the form named, and every call the form
    bq_expect_launch gives.  Measured (H100 80GB HBM3, 400 W): err_gpu at most 0.25 of its bound in every case.  The
    10 Hz / 192 kHz lowpass with Q 5 is at most 2.9e-12 relative over its inputs (the FP64 recurrence: up to 1.6e-10);
    with the scan in the companion basis (before biquad.cu's basis change) it was 1.4e-9 on the sine input."""
    sec = BQ_SECTIONS[name]
    fs = sec[1]
    coefs = _design(gpu_lib, sec)[None, :]
    N = 6 * 4096 + 1
    x = bq_inputs(fs, N, seed=len(name))
    F = 2048 if form == "split" else 4096
    ch = gpu_lib.Chain(fs, 4).add_biquad(coefs)

    def run(a, b):
        y = ch.run(x[a:b]).copy()
        d, want = ch.describe()[0], bq_expect_launch(4, 1, b - a)
        assert (d["ch"], d["split"]) == (want["ch"], want["split"]), (a, b, d)
        assert b - a != F or d["split"] == (form == "split"), (a, b, d)
        return y
    got = np.concatenate([run(i, min(i + F, N)) for i in range(0, N, F)])
    bq_check("%s/%s" % (name, form), got, x, coefs)
    ch.reset()
    cuts = [0, 1, 2047, 2049, 4096, 8192, 8193, 12287, 16384, N] if form == "split" else [0, 4095, 8191, 8192, 12289, 20000, N]
    got2 = np.concatenate([run(a, b) for a, b in zip(cuts[:-1], cuts[1:])])
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


# ------------------------------------------------------------------------------------------------------------
# Resample
# ------------------------------------------------------------------------------------------------------------
RS_RMS, RS_MAX = 1e-14, 1e-13
_G_CACHE = {}


def _table_factor(gpu_lib, fi, fo, bw):
    """max(1, sqrt(K / 8192)), K = sinc_len: what the stream bounds are multiplied by.  The device builds each tap as
    a K-term cosine sum in FP64 (k_rs_table, after a K-bin DFT of the sinc).  Its error per tap stays below 5e-15
    ||G|| (readback below), but an output sums in_len of those errors, and where they are correlated along the window
    (a sine, a DC step) they add up: the FMA and tensor-core kernels, which sum in different orders, show identical
    stream errors, so the table, not the accumulation, is what they measure.  Measured (H100 80GB HBM3, 400 W): at
    most 2.8e-15 RMS up to K = 8000; 1.0e-14 RMS / 4.6e-14 max at K = 21504 (6:1, bandwidth 0.99); 1.5e-14 / 5.9e-14
    at K = 71680 (2:1 and 1:2, bandwidth 0.999).  Up to K = 8192 (every ratio at the default bandwidth) the bounds
    apply as they are."""
    return max(1.0, np.sqrt(gpu_lib.resample_params(fi, fo, bw)["sinc_len"] / 8192.0))


def _taps(fi, fo, bw):
    if (fi, fo, bw) not in _G_CACHE:
        _G_CACHE[(fi, fo, bw)] = resample_taps_truth(fi, fo, bw)
    return _G_CACHE[(fi, fo, bw)]


def _rs_chain(gpu_lib, fi, fo, C, bw, tile=None):
    """A chain with one resampler; `tile` forces DSP_B200_RS_TILE for this operator (None: the default)."""
    with env(DSP_B200_RS_TILE=tile):
        return gpu_lib.Chain(fi, C).add_resample(fo, bw)


def _plan(ch):
    p = ch.describe()[0]
    assert p["op"] == "resample", p
    return p


def rs_bases(fi, fo, bw, N, seed):
    """[N, 5]: dyadic white noise; a 0.9 full-scale sine just inside the passband edge; a tone in the stopband (in the
    transition band when upsampling, where the input has no stopband); a DC step 0 -> 0.9; +-0.5 at the input Nyquist."""
    rng = np.random.default_rng(seed)
    t = np.arange(N) / fi
    mn = min(fi, fo)
    x = np.zeros((N, 5))
    x[:, 0] = dyadic_signal(rng, N, 1)[:, 0]
    x[:, 1] = 0.9 * np.sin(2 * np.pi * 0.97 * bw * mn / 2 * t + 0.3)
    f_stop = 0.5 * (mn / 2 + fi / 2) if fo < fi else 0.499 * fi
    x[:, 2] = 0.9 * np.sin(2 * np.pi * f_stop * t + 1.1)
    x[N // 3:, 3] = 0.9
    x[:, 4] = 0.5 * (1 - 2 * (np.arange(N) % 2))
    return x


def _tiled(base, C):
    return np.ascontiguousarray(base[:, np.arange(C) % base.shape[1]])


def _check_stream(name, got, base, fi, fo, bw, rows=None, seed=0, factor=1.0):
    """got [n_out, C] (channel c carries base c % 5): the first channels against the truth (on `rows` or, past 4000
    outputs, on the first and last 200 and a seeded sample), the others bit for bit equal to them.  Returns the errors."""
    C, k = got.shape[1], min(got.shape[1], base.shape[1])
    for c in range(k, C):
        assert np.array_equal(got[:, c], got[:, c % base.shape[1]]), (name, c)
    G = _taps(fi, fo, bw)
    if rows is None:
        rows = np.arange(got.shape[0])
        if rows.size > 4000:
            rng = np.random.default_rng(seed)
            rows = np.unique(np.concatenate([rows[:200], rows[-200:], rng.choice(rows, 3600, replace=False)]))
    want = resample_truth(base[:, :k], fi, fo, bw, got.shape[0], rows=rows, G=G)
    r, m = rs_nerr(got[rows, :k], want, base[:, :k], G)
    _record("resample", name, rms=r, max=m)
    assert r <= RS_RMS * factor and m <= RS_MAX * factor, (name, r, m, factor)
    return r, m


def _run_calls(ch, x, sizes):
    outs, pos = [], 0
    for f in sizes:
        outs.append(ch.run(x[pos:pos + f]).copy())
        pos += f
    return outs


def _drain(ch, block):
    outs = []
    while (y := ch.drain(block)) is not None:
        outs.append(y)
    return outs


RS_READBACK = [(r, bw) for bw in (0.7, 0.99) for r in [(44100, 48000), (48000, 44100), (44100, 192000), (8000, 48000),
                                                        (48000, 8000), (48000, 96000)]] + [((96000, 48000), 0.999), ((48000, 96000), 0.999)]


@pytest.mark.parametrize("rates,bw", RS_READBACK, ids=lambda v: "%d-%d" % v if isinstance(v, tuple) else "bw%s" % v)
def test_resample_tap_table_readback(gpu_lib, rates, bw):
    """Channel c carries one unit impulse, at input row r0 + c (c < d, r0 >= 2 in_len): every emitted output is then
    exactly one tap, G[(m d) mod n][floor(m d / n) - r0 - c], and every other product is an exact zero, so the d
    channels read the device's whole table back.  Each tap against the long-double table, and exactly 0.0 wherever
    the window misses the impulse; on C = d channels through the FMA kernel (DSP_B200_RS_TILE=3) and on d rounded up
    to a multiple of 4 through the tensor-core default, which must read the same bits.  Bound max |dG| <= 1e-14 ||G||
    times _table_factor."""
    fi, fo = rates
    G = _taps(fi, fo, bw)
    n, in_len = G.shape
    nG = taps_norm(G)
    p = gpu_lib.resample_params(fi, fo, bw)
    d, out_delay = p["d"], p["out_delay"]
    r0 = 2 * in_len
    N = r0 + 2 * d + in_len + 64
    got = []
    for C, tile, kernel in ((d, 3, "k_rs_poly"), (d + (-d) % 4, None, "k_rs_mma2")):
        x = np.zeros((N, C))
        x[r0 + np.arange(C), np.arange(C)] = 1.0
        ch = _rs_chain(gpu_lib, fi, fo, C, bw, tile)
        y = np.concatenate(_run_calls(ch, x, [4096] * (N // 4096) + [N % 4096]) + _drain(ch, 4096))
        assert _plan(ch)["kernel"] == kernel
        ch.close()
        m = out_delay + np.arange(y.shape[0])
        ph, ih = (m * d) % n, (m * d) // n
        t = ih[:, None] - r0 - np.arange(C)[None, :]
        inside = (t >= 0) & (t < in_len)
        cover = np.zeros((n, in_len), dtype=bool)
        cover[np.broadcast_to(ph[:, None], t.shape)[inside], t[inside]] = True
        assert cover.all(), "the impulses do not reach every tap"
        assert np.all(y[~inside] == 0.0), (C, "nonzero output where the window misses the impulse")
        want = G.astype(np.float64)[np.broadcast_to(ph[:, None], t.shape)[inside], t[inside]]
        err = float(np.max(np.abs(y[inside] - want))) / nG
        _record("resample", "readback/%d-%d/bw%s/C%d" % (fi, fo, bw, C), max=err)
        assert err <= 1e-14 * _table_factor(gpu_lib, fi, fo, bw), (C, err)
        got.append(y[:, :d])
    assert np.array_equal(got[0], got[1]), "the FMA and tensor-core kernels read different taps"


RS_SHAPES = {"mma": [4, 36, 64, 68, 124, 132, 260], "pair": [2, 66, 130], "single": [1, 33, 129]}


@pytest.mark.parametrize("shape", list(RS_SHAPES))
def test_resample_every_variant_at_channel_tile_edges(gpu_lib, shape):
    """44100 -> 48000 with DSP_B200_RS_TILE = 0 (default) and 1..7 on channel counts at the tile edges of each kernel
    (tensor-core shapes: a partly filled warp, CTA column or last 128 channels; pair and single-channel shapes for the
    FMA kernel, on which a forced tile the count cannot use falls back to the default), calls of 1, 7, in_len - 1,
    in_len, in_len + 1 and 4096 frames, then the drain.  describe() names the kernel and tile that ran; counts as
    rs_counts replays them; the five base signals against the truth, their copies in the other channels bit for bit;
    and within each family (tiles 1-3 on the FMA kernel, 4-7 on the tensor cores) every tile gives the same bits: an
    output meets the same products in the same order, and the leading zero taps add exact zeros."""
    fi, fo, bw = 44100, 48000, 0.939
    in_len = gpu_lib.resample_params(fi, fo)["in_len"]
    sizes = [1, 7, in_len - 1, in_len, in_len + 1, 4096, 1, 4096]
    N = sum(sizes)
    base = rs_bases(fi, fo, bw, N, seed=7)
    counts, drains = rs_counts(fi, fo, sizes, 1000, bw)
    worst = (0.0, 0.0)
    for C in RS_SHAPES[shape]:
        x = _tiled(base, C)
        family = {}
        for force in range(8):
            want = rs_expect_launch(C, force, 1, 1)
            tile, kernel = want["tile"], want["kernel"]
            ch = _rs_chain(gpu_lib, fi, fo, C, bw, force)
            outs = _run_calls(ch, x, sizes)
            plan = _plan(ch)
            dr = _drain(ch, 1000)
            ch.close()
            assert (plan["force_tile"], plan["tile"], plan["kernel"]) == (force, tile, kernel), (C, force, plan)
            assert [o.shape[0] for o in outs] == counts and [o.shape[0] for o in dr] == drains, (C, force)
            got = np.concatenate(outs + dr)
            fam = tile >= 4
            if fam in family:
                assert np.array_equal(got, family[fam]), (C, force, "differs from another tile of its family")
                continue
            family[fam] = got
            e = _check_stream("variants/C%d/tile%d" % (C, tile), got, base, fi, fo, bw)
            worst = (max(worst[0], e[0]), max(worst[1], e[1]))
    _record("resample", "variants/%s/worst" % shape, rms=worst[0], max=worst[1])


@pytest.mark.parametrize("C", [68, 132, 260])
def test_resample_warps_per_cta(gpu_lib, C):
    """The tensor-core kernels' warps per CTA (4, 2 or 1, from the channel count, the output tiles of the call and
    the device's SM count) on 68, 132 and 260 channels (the last 64- or 128-channel column partly filled), for tiles
    4-7, with call sizes scaled by the SM count so that each call reaches a known choice: describe() reports the
    choice resample.cu's formula makes for the frames the call emitted, and every choice the channel count allows is
    reached.  Values against the truth, copies bit for bit."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    fi, fo, bw = 44100, 48000, 0.939
    sizes = [k * sms for k in (4, 16, 26, 36, 50, 64)] + [3]
    N = sum(sizes)
    base = rs_bases(fi, fo, bw, N, seed=C)
    x = _tiled(base, C)
    allowed = {1, 2, 4} if C >= 128 else {1, 2}
    ref = None
    for force in (4, 5, 6, 7):
        ch = _rs_chain(gpu_lib, fi, fo, C, bw, force)
        outs, reached = [], set()
        pos = 0
        for f in sizes:
            outs.append(ch.run(x[pos:pos + f]).copy())
            pos += f
            if outs[-1].shape[0]:
                plan = _plan(ch)
                want = rs_expect_launch(C, force, outs[-1].shape[0], sms)
                assert (plan["tile"], plan["warps"]) == (force, want["warps"]), (force, outs[-1].shape[0], plan)
                assert plan["depth"] == want["depth"], plan
                reached.add(want["warps"])
        ch.close()
        assert reached == allowed, (force, reached)
        got = np.concatenate(outs)
        if ref is None:
            ref = got
            _check_stream("warps/C%d" % C, got, base, fi, fo, bw)
        else:
            assert np.array_equal(got, ref), force


def _rates_id(r):
    return "%d-%d" % r


@pytest.mark.parametrize("bw", [0.7, 0.99])
@pytest.mark.parametrize("rates", RS_RATIOS, ids=_rates_id)
def test_resample_ratios_and_bandwidths(gpu_lib, rates, bw):
    """The 15 ratios of test_resample_ratios at bandwidths 0.7 and 0.99 (`resample 0.99 48000`), on 5 channels (the
    FMA kernel) and 8 (tensor cores), ragged calls and the drain; counts as rs_counts replays them, the five inputs
    against the truth."""
    _ratio_case(gpu_lib, rates, bw)


@pytest.mark.parametrize("rates", [(96000, 48000), (48000, 96000)], ids=_rates_id)
def test_resample_bandwidth_0_999(gpu_lib, rates):
    """Bandwidth 0.999 at 2:1 and 1:2: in_len is tens of thousands (long k_end loops, many tap chunks, a large padded
    table) while the table itself is cheap (n <= 2); checked on a seeded sample of outputs."""
    _ratio_case(gpu_lib, rates, 0.999, sample=2000)


def _ratio_case(gpu_lib, rates, bw, sample=None):
    fi, fo = rates
    in_len = gpu_lib.resample_params(fi, fo, bw)["in_len"]
    rng = np.random.default_rng(fi + fo)
    sizes = [1, 7, in_len - 1, in_len, in_len + 1]
    while sum(sizes) < 3 * in_len + 2000:
        sizes.append(int(rng.integers(1, 4097)))
    N = sum(sizes)
    base = rs_bases(fi, fo, bw, N, seed=fi + fo)
    counts, drains = rs_counts(fi, fo, sizes, 4096, bw)
    rows, ref = None, None
    for C, kernel in ((5, "k_rs_poly"), (8, "k_rs_mma2")):
        ch = _rs_chain(gpu_lib, fi, fo, C, bw)
        outs = _run_calls(ch, _tiled(base, C), sizes)
        assert _plan(ch)["kernel"] == kernel
        dr = _drain(ch, 4096)
        ch.close()
        assert [o.shape[0] for o in outs] == counts and [o.shape[0] for o in dr] == drains, C
        got = np.concatenate(outs + dr)
        if sample and rows is None:
            rows = np.unique(np.concatenate([np.arange(100), got.shape[0] - 1 - np.arange(100),
                                             rng.choice(got.shape[0], sample, replace=False)]))
        _check_stream("ratios/%d-%d/bw%s/C%d" % (fi, fo, bw, C), got, base, fi, fo, bw, rows=rows, seed=fi,
                      factor=_table_factor(gpu_lib, fi, fo, bw))


def _pacing_to(fi, fo, bw, target, block=1000):
    """Smallest stream of `block`-frame calls (from 5 in_len on) after which in_buf_pos == target."""
    p0 = RsPacing(fi, fo, bw)
    N = 5 * p0.in_len
    while True:
        p = RsPacing(fi, fo, bw)
        sizes = [block] * (N // block) + ([N % block] if N % block else [])
        for f in sizes:
            p.run(f)
        if p.in_buf_pos == target:
            return sizes
        N += 1


@pytest.mark.parametrize("rates", [(44100, 48000), (48000, 8000)], ids=_rates_id)
@pytest.mark.parametrize("case", ["first_block", "wrap_then_grow", "reset", "drain_end", "drain_reset_drain"])
def test_resample_stream_shapes(gpu_lib, rates, case):
    """Per-call counts against rs_counts / RsPacing and values against the truth, on 5 (FMA) and 8 (tensor-core)
    channels: calls summing to in_len - 1, in_len and in_len + 1 before the first output; 2000 calls of 5 frames (the
    ring wraps many times), one of 50000 (the ring grows after a wrap) and small calls again; reset() mid-stream, then
    1 frame and 8192; the drain after streams that end with in_buf_pos = 0, in_len - 1 and mid-block, polled 1 (when
    upsampling), 7 and 4096 frames at a time; drain, reset(), the stream again, and a second drain, which is dry because the drain
    counters persist across reset() as in the reference."""
    fi, fo = rates
    bw = 0.939
    L = gpu_lib.resample_params(fi, fo)["in_len"]
    runs = []   # (name, sizes, drain poll or None); a None entry in `runs` is a reset()
    if case == "first_block":
        for k, pre in enumerate(([L - 1], [L - 3, 2], [L], [L - 1, 1], [L + 1], [1, L - 1, 1])):
            runs.append([("pre%d" % k, pre + [7, L, 4096, 1], 4096)])
    elif case == "wrap_then_grow":
        runs.append([("wrap_grow", [5] * 2000 + [50000] + [3] * 300, None)])
    elif case == "reset":
        runs.append([("before", [1000] * 3 + [L // 2], None), None, ("after", [1, 8192], 7)])
    elif case == "drain_end":
        for target in (0, L - 1, L // 2):
            for poll in (1, 7, 4096) if fo > fi else (7, 4096):   # 1-frame polls at 6:1: mostly empty host calls
                runs.append([("end%d/poll%d" % (target, poll), _pacing_to(fi, fo, bw, target), poll)])
    else:
        runs.append([("first", [3000, 1, 2000], 1000), None, ("again", [2500, 4096], 1000)])
    for C in (5, 8):
        for seq in runs:
            ch = _rs_chain(gpu_lib, fi, fo, C, bw)
            pacing = RsPacing(fi, fo, bw)
            for step in seq:
                if step is None:
                    ch.reset()
                    pacing.reset()
                    continue
                name, sizes, poll = step
                N = sum(sizes)
                base = rs_bases(fi, fo, bw, N, seed=N + C)
                outs = _run_calls(ch, _tiled(base, C), sizes)
                assert [o.shape[0] for o in outs] == [pacing.run(f) for f in sizes], name
                if poll:
                    dr = _drain(ch, poll)
                    want = []
                    while (o := pacing.drain(poll)) is not None:
                        want.append(o)
                    assert [o.shape[0] for o in dr] == want, name
                    outs += dr
                got = np.concatenate(outs)
                if case == "drain_reset_drain" and name == "again":
                    assert want == [], "the second drain after reset() must be dry"
                if got.shape[0]:
                    _check_stream("stream/%d-%d/%s/%s/C%d" % (fi, fo, case, name, C), got, base, fi, fo, bw)
            ch.close()
