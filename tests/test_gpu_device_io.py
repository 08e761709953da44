"""GPU tier: device-resident calls (run_device) on the caller's buffers and on the caller's streams.

In Mode D the caller owns the input rows, the output rows and the stream.  The header asks no more of them than
device-resident interleaved doubles (8-byte alignment) and any stream, so these tests do what a caller may do.

Footprint and alignment (test_*_footprint): every call gets one fresh device tensor [guard | input rows | guard |
output rows (max_out_frames) | guard] filled with a NaN canary, with d_in and d_out each at a 16-byte-aligned offset or
one double past it (four layouts) and, where the chain allows it, in place one double past an aligned offset.  After
each call the guards and the output rows at and past the returned frame count still hold the canary, d_in holds its
input bit for bit (out of place), and the output is bit-identical, call by call, to the same chain run in host mode
(aligned buffers of the library's own); the host-mode run is checked against the extended-precision truths of
tests/accuracy.py.  Resample on 1, 2, 6, 36, 68, 132 and 260 channels with every DSP_B200_RS_TILE each count allows:
k_rs_poly with 1, 2 and 4 channels per lane, k_rs_mma and k_rs_mma2 (the 4096-frame call reaches 4 warps per CTA on 260
channels, 2 on 68 and 132 and 1 on 36 on a 132-SM H100); misaligned outputs report out_align 8.  FIR: one case of every
FIR_CASES family, the full-wave plan with its mid-window pass, the far-tier edge far/P48, the latency ring and a
scattered selector; on misaligned rows the fused kernel's cluster form (128-bit row accesses) is never taken.

The caller's streams (test_*_caller_streams): the chains A, B and C of test_gpu_chain on their one- and several-slab
layouts, shard by shard, and the FIR cases that run work on the library's side streams, on a new non-blocking stream,
on the legacy stream, alternating between two non-blocking streams (the caller orders them with an event after every
call), and with ONE d_in / d_out pair reused for every call: before each call the caller's stream spins (a bounded
torch.cuda._sleep), then copies the next block into d_in; after it, d_out is copied into a history tensor and d_in is
filled with NaN, with no host synchronisation until the end.  A launch that does not wait for the caller's earlier work
reads a stale or NaN block, and one the caller's stream does not wait for is missed by the history copy, so the
history must be bit-identical to host mode and free of NaN whatever the timing.

The whole file takes about 25 s (measured on an H100 80GB HBM3 at its 700 W limit).
"""
import functools
import zlib

import numpy as np
import pytest

from accuracy import FIR_CASES, FIR_EDGES, biquad_within_ref, dyadic_signal, env, exact_conv, fir_nerr, rs_counts, rs_expect_launch
from test_gpu_accuracy import (BQ_SECTIONS, FIR_MAX, FIR_RMS, H_SHIFT, _check_plan, _check_stream, _design,
                               _rs_chain, _run_calls, _tiled, bq_inputs, ir_family, rs_bases)
from test_gpu_chain import _add_ops, _inputs as chain_inputs, _op_index, _reference as chain_reference, _same, _spec as chain_spec
from test_gpu_fir_full_wave import full_wave_channels

pytestmark = pytest.mark.gpu

CANARY = 0x7FF80000DEADBEEF      # a quiet NaN with a payload no kernel computes
GUARD = 8                         # doubles before, between and after the caller's rows (even: keeps offsets 16-byte aligned)
# (d_in one double past a 16-byte-aligned offset, d_out one double past, in place)
LAYOUTS = [(0, 0, False), (1, 0, False), (0, 1, False), (1, 1, False)]
IN_PLACE = (1, 1, True)
SLEEP_CYCLES = 200000             # torch.cuda._sleep before each call of the reuse mode: about 0.1 ms
MODES = ["stream", "legacy", "alternate", "reuse"]


def _layout_id(layout):
    return "in_place" if layout[2] else "in%d_out%d" % (8 * layout[0] + 8, 8 * layout[1] + 8)


def _footprint_run(ch, x_dev, sizes, C, layout, op_index=None):
    """The calls of `sizes` frames (x_dev: the stream [N, C] on the device), each on a fresh canary-filled caller tensor
    in `layout`, on the legacy stream.  Asserts the footprint; returns the outputs per call (numpy) and describe() of
    operator `op_index` after each call."""
    import torch
    in_odd, out_odd, in_place = layout
    outs, flags, plans, pos = [], [], [], 0
    for f in sizes:
        mo = ch.max_out_frames(f)
        i0 = GUARD + in_odd
        i1 = i0 + f * C
        o0 = i0 if in_place else (i1 + GUARD + 1) // 2 * 2 + out_odd
        o1 = o0 + (max(mo, f) if in_place else mo) * C
        buf = torch.empty(o1 + GUARD, dtype=torch.float64, device="cuda")
        bits = buf.view(torch.int64)
        bits.fill_(CANARY)
        xin = x_dev[pos:pos + f].reshape(-1)
        buf[i0:i1] = xin
        assert ((buf.data_ptr() + 8 * i0) % 16, (buf.data_ptr() + 8 * o0) % 16) == (8 * in_odd, 8 * (in_odd if in_place else out_odd))
        n = ch.run_device(0, f, buf.data_ptr() + 8 * i0, buf.data_ptr() + 8 * o0, None)
        end = o0 + n * C
        changed = bits != CANARY
        # the guard and canary rows outside [d_out, d_out + n rows), and (out of place) the input rows
        outside = changed[:i0].any() | changed[end:].any() | (changed[i1:o0].any() if not in_place else False)
        inp = (bits[i0:i1] != xin.view(torch.int64)).any() if not in_place else torch.zeros((), dtype=torch.bool, device="cuda")
        flags.append(torch.stack([outside, inp]))
        outs.append(buf[o0:end].view(n, C).clone())
        if op_index is not None:
            plans.append(ch.describe()[op_index])
        pos += f
    torch.cuda.synchronize()
    for i, (outside, inp) in enumerate(torch.stack(flags).cpu().numpy()):
        assert not outside, (_layout_id(layout), "call %d wrote outside its returned output rows" % i, sizes[i])
        assert not inp, (_layout_id(layout), "call %d changed its input rows" % i, sizes[i])
    return [o.cpu().numpy() for o in outs], plans


# ------------------------------------------------------------------------------------------------------------
# footprint and alignment: resample
# ------------------------------------------------------------------------------------------------------------
RS_FI, RS_FO, RS_BW = 44100, 48000, 0.939


@pytest.mark.parametrize("C", [1, 2, 6, 36, 68, 132, 260])
def test_resample_footprint(gpu_lib, C):
    """44100 -> 48000, calls of 1, 7, in_len - 1, in_len, in_len + 1 and 4096 frames, every DSP_B200_RS_TILE the
    channel count allows, in the four layouts: counts as rs_counts replays them, describe() names the tile, kernel,
    warps and out_align (8 exactly when d_out is misaligned) of each call that emitted frames, and every layout is
    bit-identical to host mode; the host-mode stream against the long-double truth (once per kernel family: the tiles
    of a family agree bit for bit)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    in_len = gpu_lib.resample_params(RS_FI, RS_FO)["in_len"]
    sizes = [1, 7, in_len - 1, in_len, in_len + 1, 4096]
    base = rs_bases(RS_FI, RS_FO, RS_BW, sum(sizes), seed=C)
    x = _tiled(base, C)
    x_dev = torch.from_numpy(x).cuda()
    counts, _ = rs_counts(RS_FI, RS_FO, sizes)
    tiles = {}
    for force in range(8):
        tiles.setdefault(rs_expect_launch(C, force, 1, sms)["tile"], force)
    family = {}
    for tile, force in sorted(tiles.items()):
        kernel = rs_expect_launch(C, force, 1, sms)["kernel"]
        ch = _rs_chain(gpu_lib, RS_FI, RS_FO, C, RS_BW, force)
        want = _run_calls(ch, x, sizes)
        ch.close()
        assert [w.shape[0] for w in want] == counts, (C, tile)
        whole = np.concatenate(want)
        fam = tile >= 4
        if fam in family:
            assert np.array_equal(whole, family[fam]), (C, tile, "differs from another tile of its family")
        else:
            family[fam] = whole
            _check_stream("device_io/C%d/tile%d" % (C, tile), whole, base, RS_FI, RS_FO, RS_BW)
        for layout in LAYOUTS:
            ch = _rs_chain(gpu_lib, RS_FI, RS_FO, C, RS_BW, force)
            got, plans = _footprint_run(ch, x_dev, sizes, C, layout, op_index=0)
            ch.close()
            for k, p in enumerate(plans):
                if counts[k] == 0:
                    continue
                warps = rs_expect_launch(C, force, counts[k], sms)["warps"]
                assert (p["tile"], p["kernel"], p["warps"], p["out_align"]) == (tile, kernel, warps, 8 if layout[1] else 16), (C, layout, k, p)
            _same(got, want, "C%d tile %d %s vs host mode" % (C, tile, _layout_id(layout)))


@pytest.mark.parametrize("C", [6, 8])
def test_biquad_resample_chain_footprint(gpu_lib, C):
    """biquad -> resample 44100 -> 48000 (the resampler writes the caller's rows from the chain's own scratch rows) on
    6 channels (channel pairs) and 8 (tensor cores), in the four layouts: bit-identical to host mode, out_align 8 on a
    misaligned d_out."""
    import torch
    fs = RS_FI
    coefs = np.array([gpu_lib.biquad_design(13, fs, f, q, g) for f, q, g in ((200.0, 0.9, 6.0), (3000.0, 1.3, -3.0))])
    sizes = [1000, 1, 4096, 587, 4097, 20000, 3]
    x = np.random.default_rng(C).standard_normal((sum(sizes), C)) * 0.2
    x_dev = torch.from_numpy(x).cuda()

    def chain():
        return gpu_lib.Chain(fs, C).add_biquad(coefs).add_resample(RS_FO)
    ch = chain()
    want = _run_calls(ch, x, sizes)
    ch.close()
    assert sum(w.shape[0] for w in want) > 30000
    for layout in LAYOUTS:
        ch = chain()
        got, plans = _footprint_run(ch, x_dev, sizes, C, layout, op_index=1)
        ch.close()
        assert all(p["out_align"] == (8 if layout[1] else 16) for p, w in zip(plans, want) if w.shape[0]), (layout, plans)
        assert plans[-1]["kernel"] == ("k_rs_poly" if C % 4 else "k_rs_mma2"), plans[-1]
        _same(got, want, "biquad -> resample, C%d %s vs host mode" % (C, _layout_id(layout)))


# ------------------------------------------------------------------------------------------------------------
# footprint and alignment: biquad, gain, align
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [3, 257])
@pytest.mark.parametrize("call", [2048, 4097])
def test_biquad_footprint(gpu_lib, C, call):
    """Two ill-conditioned sections at 192 kHz, calls of 2048 frames (the split form: two CTAs per channel pair) or
    4097 (the 16-warp form), 3 and 257 channels, in the four layouts and in place: bit-identical to host mode, and
    host mode within biquad_within_ref of the long-double cascade."""
    import torch
    fs = 192000
    coefs = np.array([_design(gpu_lib, BQ_SECTIONS[n]) for n in ("lowpass_10_192k_q5", "notch_10_192k_q10")])
    sizes = [call] * 3 + [5]
    base = bq_inputs(fs, sum(sizes), seed=C + call)
    x = np.ascontiguousarray(np.tile(base, (1, (C + 3) // 4))[:, :C])
    x_dev = torch.from_numpy(x).cuda()
    ch = gpu_lib.Chain(fs, C).add_biquad(coefs)
    want = _run_calls(ch, x, sizes)
    ch.close()
    host = np.concatenate(want)
    k = min(C, 4)
    biquad_within_ref(host[:, :k], base[:, :k], coefs)
    for c in range(4, C):
        assert np.array_equal(host[:, c], host[:, c % 4]), c
    for layout in LAYOUTS + [IN_PLACE]:
        ch = gpu_lib.Chain(fs, C).add_biquad(coefs)
        got, _ = _footprint_run(ch, x_dev, sizes, C, layout)
        ch.close()
        _same(got, want, "biquad C%d call %d %s vs host mode" % (C, call, _layout_id(layout)))


def test_gain_footprint(gpu_lib):
    """gain with mult and add on dyadic values (x mult + add is exact, so the fused multiply-add must give it exactly),
    in the four layouts and in place."""
    import torch
    C = 7
    sizes = [1, 100, 4096, 4097, 3]
    x = dyadic_signal(np.random.default_rng(7), sum(sizes), C)
    mult = (np.arange(C) - 3) / 64.0 + 0.75
    add = (np.arange(C) - 2) / 256.0
    x_dev = torch.from_numpy(x).cuda()
    truth = x * mult + add
    for layout in LAYOUTS + [IN_PLACE]:
        ch = gpu_lib.Chain(48000, C).add_gain(mult, add)
        got, _ = _footprint_run(ch, x_dev, sizes, C, layout)
        ch.close()
        assert [g.shape[0] for g in got] == sizes
        assert np.array_equal(np.concatenate(got), truth), _layout_id(layout)


def test_align_footprint(gpu_lib):
    """align with per-channel delays (0 .. 5000 frames) and a 1000-frame discard, so that the first calls return fewer
    rows than they were given (none, then part of a block): in the four layouts, the delayed stream exactly."""
    import torch
    C = 6
    delays = [0, 1, 700, 5000, 3, 0]
    sizes = [1, 7, 600, 4096, 4097, 3, 2000]
    N = sum(sizes)
    x = np.random.default_rng(11).standard_normal((N, C))
    x_dev = torch.from_numpy(x).cuda()
    truth = np.zeros_like(x)
    for c, d in enumerate(delays):
        truth[d:, c] = x[:N - d, c]
    truth = truth[1000:]
    cum = np.cumsum(sizes)
    want_counts = list(np.diff(np.concatenate([[0], np.maximum(cum - 1000, 0)])))
    assert want_counts[:3] == [0, 0, 0] and 0 < want_counts[3] < sizes[3]
    for layout in LAYOUTS:
        ch = gpu_lib.Chain(48000, C).add_align(delays, 1000)
        got, _ = _footprint_run(ch, x_dev, sizes, C, layout)
        ch.close()
        assert [g.shape[0] for g in got] == want_counts, (_layout_id(layout), [g.shape[0] for g in got])
        assert np.array_equal(np.concatenate(got), truth), _layout_id(layout)


# ------------------------------------------------------------------------------------------------------------
# footprint and alignment: FIR
# ------------------------------------------------------------------------------------------------------------
FIR_IO = ["multi_300", "single_4096_t8", "merge", "pipe_4096", "bulk_32768", "far/P48", "full_wave_pass", "latency", "scattered"]
FIR_SIDE = ["multi_300", "single_4096_t8", "merge", "pipe_4096", "full_wave_pass", "far/P48"]


def _fir_sizes(frames, N):
    """Whole calls, a ragged pair that ends on a block boundary again, whole calls, the remainder."""
    sizes = [frames] * 4 + [frames // 2 - 3, frames // 2 + 3]
    sizes += [frames] * ((N - sum(sizes)) // frames)
    return sizes + ([N - sum(sizes)] if N > sum(sizes) else [])


@functools.lru_cache(maxsize=None)
def _fir_case(case):
    """(C, taps h, selector, latency, block hint, envs, call sizes, x, plan check) of a FIR case."""
    sel, lat = None, 0
    if case in FIR_CASES:
        frames, taps, C, hint, envs, check = FIR_CASES[case]
    elif case == "far/P48":
        e = FIR_EDGES[case]
        frames, taps, C, hint, envs = e["hint"], e["taps"], e["C"], e["hint"], e["envs"]
        check = functools.partial(_check_plan, want=e["plan"], case=case)
    elif case == "full_wave_pass":
        frames, taps, C, hint, envs = 4096, 131072, None, 4096, {}
        check = lambda p: (p["levels"] == [{"B": 4096, "P": 32}] and p["lookahead"] == 2 and p["pass_m"] > 0)
    else:
        frames, taps, C, hint, envs = 4096, 40000, (8 if case == "latency" else 12), 4096, {}
        lat = 24576 if case == "latency" else 0
        if case == "scattered":
            sel = tuple(c in (1, 2, 3, 5, 6, 7, 10, 11) for c in range(C))
        check = lambda p: len(p["levels"]) == 1
    if C is None:
        C = full_wave_channels(4096)
    n_sel = C if sel is None else sum(sel)
    N = taps + 4 * max(frames, 4096) + 77
    rng = np.random.default_rng(zlib.crc32(b"device_io" + case.encode()))
    h = ir_family("comb", taps, n_sel, seed=taps)
    x = dyadic_signal(rng, N, C)
    return C, h, sel, lat, hint, envs, _fir_sizes(frames, N), x, check


def _fir_chain(gpu_lib, case):
    C, h, sel, lat, hint, envs, _, _, _ = _fir_case(case)
    with env(**envs):
        return gpu_lib.Chain(48000, C).add_fir(h, selector=sel, latency=lat, block_hint=hint)


@functools.lru_cache(maxsize=None)
def _fir_host(gpu_lib, case):
    """Host mode: the outputs per call and the plan, checked against the exact convolution (on at most eight channels)."""
    C, h, sel, lat, hint, envs, sizes, x, check = _fir_case(case)
    with env(**envs):
        ch = _fir_chain(gpu_lib, case)
        want = _run_calls(ch, x, sizes)
        plan = ch.describe()[0]
    ch.close()
    ok = check(plan)   # _check_plan asserts, the FIR_CASES checks return a bool
    assert ok is None or ok, (case, plan)
    got = np.concatenate(want)
    cols = [c for c in range(C) if sel is None or sel[c]]
    pick = sorted(set(cols[:4] + cols[-4:]))
    hk = h[:, [cols.index(c) for c in pick]]
    exact = exact_conv(x[:, pick], hk, H_SHIFT, latency=lat)
    r, m = fir_nerr(got[:, pick], exact, x[:, pick], hk)
    assert r <= FIR_RMS and m <= FIR_MAX, (case, r, m, plan)
    for c in range(C):
        if sel is not None and not sel[c]:
            assert np.array_equal(got[:, c], x[:, c]), (case, c)
    return want, plan


@pytest.mark.parametrize("case", FIR_IO)
def test_fir_footprint(gpu_lib, case):
    """One case of every FIR_CASES family (multi-level with the head kernel and k_fir_unstash, the folded fused kernel,
    the merged MAC grid, the pipeline kernel, the bulk form's scatter), the full-wave plan with its mid-window pass, the
    far-tier edge far/P48, the latency ring (k_delay_read) and a scattered selector, in the four layouts and in place:
    bit-identical to host mode (which matches the exact convolution), with host mode's paths, except that where the
    fused kernel meets a misaligned caller row the cluster form hands its blocks to the per-channel form."""
    import torch
    C, h, sel, lat, hint, envs, sizes, x, check = _fir_case(case)
    want, hplan = _fir_host(gpu_lib, case)
    x_dev = torch.from_numpy(x).cuda()
    hp = hplan["paths"]
    for layout in LAYOUTS + [IN_PLACE]:
        with env(**envs):
            ch = _fir_chain(gpu_lib, case)
            got, _ = _footprint_run(ch, x_dev, sizes, C, layout)
            p = ch.describe()[0]["paths"]
        ch.close()
        _same(got, want, "%s %s vs host mode" % (case, _layout_id(layout)))
        # the fused kernel reads the caller's input rows and, without a latency ring, writes the caller's output rows
        if layout[0] or (layout[1] and not lat):
            assert p == dict(hp, cluster=0, fused=hp["fused"] + hp["cluster"]), (case, _layout_id(layout), p, hp)
        else:
            assert p == hp, (case, _layout_id(layout), p, hp)
    del x_dev


def test_fir_footprint_covers_the_cluster_form(gpu_lib):
    """The cases above that run whole aligned blocks of four contiguous channels take the cluster form in host mode
    (so that the fall-back above is tested), and the others cover the pipeline, bulk and general paths."""
    used = {case: _fir_host(gpu_lib, case)[1]["paths"] for case in FIR_IO}
    for case in ("single_4096_t8", "merge", "far/P48", "full_wave_pass", "latency"):
        assert used[case]["cluster"] > 0, (case, used[case])
    assert used["pipe_4096"]["pipe"] > 0 and used["bulk_32768"]["bulk"] > 0 and used["multi_300"]["head"] > 0, used


# ------------------------------------------------------------------------------------------------------------
# the caller's streams
# ------------------------------------------------------------------------------------------------------------
def _drive(ch, xs, mode):
    """run_device on every shard of `ch` for each block of xs in one of MODES; returns the outputs per call (numpy, the
    shards' channels side by side) once the device is idle."""
    import torch
    shards = [ch.shard_info(s) for s in range(ch.n_shards)]
    max_in = max(x.shape[0] for x in xs)
    max_out = max(ch.max_out_frames(x.shape[0]) for x in xs)
    counts, keep = [], []
    if mode == "reuse":
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            xdev = [torch.from_numpy(np.ascontiguousarray(np.concatenate(xs)[:, b:b + n])).cuda() for _, b, n in shards]
            d_in = [torch.full((max_in, n), float("nan"), dtype=torch.float64, device="cuda") for _, _, n in shards]
            d_out = [torch.empty((max_out, n), dtype=torch.float64, device="cuda") for _, _, n in shards]
            hist = [torch.full((sum(ch.max_out_frames(x.shape[0]) for x in xs), n), float("nan"), dtype=torch.float64, device="cuda")
                    for _, _, n in shards]
            pos_in = pos_out = 0
            for x in xs:
                f = x.shape[0]
                got = set()
                for k in range(len(shards)):
                    torch.cuda._sleep(SLEEP_CYCLES)
                    d_in[k][:f].copy_(xdev[k][pos_in:pos_in + f])
                    m = ch.run_device(k, f, d_in[k].data_ptr(), d_out[k].data_ptr(), s.cuda_stream)
                    hist[k][pos_out:pos_out + m].copy_(d_out[k][:m])
                    d_in[k].fill_(float("nan"))
                    got.add(m)
                assert len(got) == 1, ("shards disagree on the frame count", got)
                m = got.pop()
                counts.append(m)
                pos_in += f
                pos_out += m
        torch.cuda.synchronize()
        h = np.concatenate([t[:pos_out].cpu().numpy() for t in hist], axis=1)
        return np.split(h, np.cumsum(counts)[:-1]) if counts else []
    if mode == "alternate":
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    elif mode == "stream":
        streams = [torch.cuda.Stream()]
    else:
        streams = [torch.cuda.default_stream()]
    ev = None
    calls = []
    for i, x in enumerate(xs):
        s = streams[i % len(streams)]
        handle = None if mode == "legacy" else s.cuda_stream
        with torch.cuda.stream(s):
            if ev is not None:
                s.wait_event(ev)
            f = x.shape[0]
            parts, got = [], set()
            for k, (_, b, n) in enumerate(shards):
                d_in = torch.from_numpy(np.ascontiguousarray(x[:, b:b + n])).cuda()
                d_out = torch.empty((max(ch.max_out_frames(f), 1), n), dtype=torch.float64, device="cuda")
                got.add(ch.run_device(k, f, d_in.data_ptr(), d_out.data_ptr(), handle))
                parts.append(d_out)
                keep.append(d_in)
            if mode == "alternate":
                ev = s.record_event()
        assert len(got) == 1, ("shards disagree on the frame count", got)
        calls.append((got.pop(), parts))
    torch.cuda.synchronize()
    return [np.concatenate([p[:m].cpu().numpy() for p in parts], axis=1) for m, parts in calls]


def _no_nan(got, what):
    for i, y in enumerate(got):
        assert not np.isnan(y).any(), (what, "NaN in call %d" % i)


CHAIN_LAYOUTS = [("A", 7, 1), ("A", 7, 3), ("B", 7, 1), ("B", 7, 3), ("C", None, 1), ("C", None, 2)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name,C,slabs", CHAIN_LAYOUTS, ids=["%s-%sch-%dslab" % (n, C or "fw", s) for n, C, s in CHAIN_LAYOUTS])
def test_chain_caller_streams(gpu_lib, name, C, slabs, mode):
    """test_gpu_chain's chains A, B and C, shard by shard, in each caller-stream mode: the per-call frame counts and
    outputs bit-identical to host mode (the pipeline of one-operator chains, itself bit-identical to the composed chain
    in host mode), no NaN, and every FIR's paths as in host mode."""
    C = C or full_wave_channels(4096)
    fs, ops = chain_spec(gpu_lib, name, C)
    ref = chain_reference(gpu_lib, name, C, slabs)
    ch = _add_ops(gpu_lib.Chain(fs, C, slabs_per_device=slabs), ops)
    try:
        got = _drive(ch, chain_inputs(name, C), mode)
        what = "%s/%d slabs/%s" % (name, slabs, mode)
        _no_nan(got, what)
        _same(got, ref["stream"], what)
        desc = ch.describe()
        assert [desc[i]["paths"] for i in _op_index(ops, ref["n_ops"])] == ref["paths"], what
    finally:
        ch.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", FIR_SIDE)
def test_fir_caller_streams(gpu_lib, case, mode):
    """The FIR plans that run work on the library's side streams (upper levels, the per-block MAC, the batch and far
    tiers, the merged grid, the pipeline kernel's batch share, the full-wave plan's pass and its fused kernel on the
    high-priority stream) in each caller-stream mode: bit-identical to host mode, no NaN, host mode's paths."""
    C, h, sel, lat, hint, envs, sizes, x, check = _fir_case(case)
    want, hplan = _fir_host(gpu_lib, case)
    xs = np.split(x, np.cumsum(sizes)[:-1])
    with env(**envs):
        ch = _fir_chain(gpu_lib, case)
        try:
            got = _drive(ch, xs, mode)
            paths = ch.describe()[0]["paths"]
        finally:
            ch.close()
    _no_nan(got, (case, mode))
    _same(got, want, "%s/%s" % (case, mode))
    assert paths == hplan["paths"], (case, mode, paths, hplan["paths"])
