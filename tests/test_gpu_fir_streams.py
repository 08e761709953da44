"""GPU tier: the FIR's cross-stream schedule under injected stream stalls.

A K2 block is spread over up to four streams: the caller's (stash, block kernel, unstash), the side stream (the upper
levels' partition-0 kernels, the per-block tail MAC), the second side stream (the batch tiers) and the look-ahead stream
of the block kernel.  Events order them and buffers are reused in rings (Y spectra, V slots, FDL rows, `pend`).  On an
idle H100 the side streams usually finish long before anyone reads their results, so a missing wait would pass every
other test.  dspb200_debug_stall() delays one stream before its first FIR launch of selected blocks, so that it falls
behind the others by several block periods:

  - each stream the plan uses, on every block (the caller's stream alone: readers lag behind writers);
  - the batch-tier stream on one block in T (each phase: one launch late by more than its ring of 2 T V slots);
  - the side stream on odd and on even blocks (the parity of the per-block MAC's two Y spectra and their events).

Stalls last 3 block times of the case, measured (2 T + 1 periods of the last level on the batch tiers' stream at
period T), within 50 us .. 5 ms.  Every case runs in host mode (Chain.run) and device-resident mode (run_device on a
caller stream); the unstalled run must match the exact convolution and a second unstalled run bit for bit, and every
stalled run must be bit-identical to it with the same describe(): a stall changes the timing only, so any difference is
a stale read.  The stall kernels are counted and timed with the profiler's event brackets, so a pattern that delays
nothing fails too.  The file takes about 4 minutes on an H100 80GB HBM3 (700 W limit).
"""
import contextlib
import time
import zlib

import numpy as np
import pytest

from accuracy import F2, F4, FIR_CASES, FIR_EDGES, FOLD_CASES, PASS_CASES, dyadic_signal, env, exact_conv, fir_nerr
from test_gpu_accuracy import FIR_MAX, FIR_RMS, H_SHIFT, _check_plan, ir_family
from test_gpu_fir_full_wave import full_wave_channels
from test_gpu_parity import eq_coefs

pytestmark = pytest.mark.gpu

MAIN, SIDE, SIDE2, HOT = 1, 2, 4, 8
ROLE_NAMES = {MAIN: "main", SIDE: "side", SIDE2: "side2", HOT: "hot"}
STALL_MIN_US, STALL_MAX_US = 50, 5000


def _case(taps, C, hint, envs=None, call=None, sel=None, latency=0, check=None, full_wave=False):
    return dict(taps=taps, C=C, hint=hint, envs=envs or {}, call=call or hint, sel=sel, latency=latency, check=check,
                full_wave=full_wave)


# Every FIR_CASES family with a side stream (multi-level, single level with tail and tiers, far tiers, the merged grid),
# the pipeline kernel and the bulk form (the caller's stream only), the FIR_EDGES groups with a side stream, every
# FOLD_CASES and PASS_CASES entry (PASS_CASES' default depth is the full-wave plan).
STREAM_CASES = {}
for _n in ("multi_64", "multi_300", "multi_1000", "single_4096_t4", "single_2048_t8", "merge", "far8_s", "far8_u", "far8_u2",
           "far16_s", "pipe_4096", "bulk_32768"):
    _frames, _taps, _C, _hint, _envs, _chk = FIR_CASES[_n]
    STREAM_CASES["paths/" + _n] = _case(_taps, _C, _hint or _frames, _envs, call=_frames, check=_chk)
for _n in ("tail/B2048_P3", "tail/B4096_P11", "tail/B2048_P22", "far/P48", "depth/T8_P19", "pipe/B2048_P11", "multi/B64_T8193",
           "multi/B256_T40961", "cluster/B4096_P3_sel2-9of10", "latency/B64_T255_lat65"):
    _e = FIR_EDGES[_n]
    STREAM_CASES["edges/" + _n] = _case(_e["taps"], _e["C"], _e["hint"], _e["envs"], call=_e["call"], sel=_e["sel"],
                                        latency=_e["latency"], check=(lambda want, n: lambda p: _check_plan(p, want, n) is None)(_e["plan"], _n))
for _n, (_taps, _C, _B, _envs, _want) in FOLD_CASES.items():
    STREAM_CASES["fold/" + _n] = _case(_taps, _C, _B, dict(_envs, DSP_B200_FIR_FOLD=1),
                                       check=(lambda w: lambda p: p["levels"][0]["P"] == w["P"] and all(p[k] == w[k] for k in ("t_batch", "t_far", "stagger")))(_want))
for _n, (_taps, _B, _P, _envs, _T, _m) in PASS_CASES.items():
    STREAM_CASES["pass/" + _n] = _case(_taps, None, _B, dict(_envs, DSP_B200_FIR_PASS=_m) if _m is not None else _envs, full_wave=True,
                                       check=(lambda P, T, m: lambda p: p["levels"][0]["P"] == P and p["t_batch"] == T and p["lookahead"] == 2
                                              and p["pass_m"] == (T // 2 if m is None else m))(_P, _T, _m))


@contextlib.contextmanager
def stalled(gpu_lib, roles, us, period=1, phase=0):
    gpu_lib.debug_stall(roles, us, period, phase)
    try:
        yield
    finally:
        gpu_lib.debug_stall(0)


def _roles(plan, device):
    """The streams a plan enqueues FIR launches on (fir.cu: advance_upper_levels, advance_tail0, launch_tail, run)."""
    multi = len(plan["levels"]) > 1
    tail0 = not multi and plan["tail_pf"] == 2 and not plan["pipe"]
    fold = tail0 and plan["l0_parts"] > 2
    roles = [MAIN]
    if multi or (tail0 and not fold):
        roles.append(SIDE)
    if plan["t_batch"] > 0 and (multi or tail0) and not plan["merge"]:
        roles.append(SIDE2)
    if tail0 and device:
        roles.append(HOT)
    return roles


def _patterns(plan, device):
    """(roles, period, phase, stall in block times), period, phase and times in level-0 blocks: each role on every block
    (3 block times); the batch tiers' stream on one block in T of the last level, at each phase that has a tier launch
    ((2 T + 1) r block times: later than its ring of 2 T V slots lasts).  The launch after last-level block q is made when level-0 block (q + 1) r
    - 1 completes, r = B_last / B0, on every q when staggered, else on q = 0 mod T.  The per-block MAC's stream on odd
    and on even blocks (3 block times)."""
    roles = _roles(plan, device)
    pats = [(r, 1, 0, 3) for r in roles]
    if SIDE2 in roles:
        T, r = plan["t_batch"], plan["levels"][-1]["B"] // plan["levels"][0]["B"]
        pats += [(SIDE2, T * r, (k + 1) * r - 1, (2 * T + 1) * r) for k in (range(T) if plan["stagger"] else [0])]
    if SIDE in roles and len(plan["levels"]) == 1:
        pats += [(SIDE, 2, 0, 3), (SIDE, 2, 1, 3)]
    return pats


class Runner:
    """One case's input through fresh chains, whole calls of `call` frames, in host mode or through run_device on a
    caller stream (torch); -> (output, describe(), seconds)."""

    def __init__(self, gpu_lib, c, x, h):
        self.gpu_lib, self.c, self.x, self.h = gpu_lib, c, x, h
        self.N = x.shape[0]
        self.d_x = self.d_y = None

    def chain(self):
        c, h = self.c, self.h
        return self.gpu_lib.Chain(48000, self.x.shape[1]).add_fir(h if h.shape[1] > 1 else h[:, 0], selector=c["sel"], latency=c["latency"],
                                                                   block_hint=c["hint"])

    def run(self, device):
        import torch
        c, x, call = self.c, self.x, self.c["call"]
        with env(**c["envs"]):
            ch = self.chain()
            if device:
                if self.d_x is None:
                    self.d_x = torch.from_numpy(x.reshape(-1)).cuda()
                    self.d_y = torch.empty_like(self.d_x)
                    self.stream = torch.cuda.Stream()
                self.d_y.fill_(np.nan)
                torch.cuda.synchronize()
                st, C = self.stream.cuda_stream, x.shape[1]
                t0 = time.perf_counter()
                for a in range(0, self.N, call):
                    assert ch.run_device(0, call, self.d_x.data_ptr() + 8 * a * C, self.d_y.data_ptr() + 8 * a * C, st) == call
                ch.join(0, st)
                self.stream.synchronize()
                dt = time.perf_counter() - t0
                got = self.d_y.cpu().numpy().reshape(x.shape)
            else:
                t0 = time.perf_counter()
                got = np.concatenate([ch.run(x[a:a + call]).copy() for a in range(0, self.N, call)])
                dt = time.perf_counter() - t0
            plan = ch.describe()[0]
        ch.close()
        return got, plan, dt


def _first_diff(got, want, B0):
    bad = np.nonzero(np.any(got != want, axis=1) & ~(np.isnan(got).all(axis=1) & np.isnan(want).all(axis=1)))[0]
    if bad.size == 0:
        return None
    f = int(bad[0])
    return dict(frame=f, block=f // B0, frames_differing=int(bad.size), max_abs=float(np.nanmax(np.abs(got - want))))


@pytest.mark.parametrize("mode", ["host", "device"])
@pytest.mark.parametrize("case", list(STREAM_CASES))
def test_fir_streams_bit_identical_under_stalls(gpu_lib, case, mode):
    """The unstalled run is exact and reproducible; every stall pattern (_patterns) gives the same bits and the same
    describe(), and its stall kernels ran for their requested time."""
    c = dict(STREAM_CASES[case])
    device = mode == "device"
    if c["full_wave"]:
        c["C"] = full_wave_channels(c["hint"])
    T, C, sel = c["taps"], c["C"], c["sel"]
    n_sel = C if sel is None else sum(sel)
    rng = np.random.default_rng(zlib.crc32(("streams" + case).encode()))
    h = ir_family("comb", T, n_sel, seed=T + 5)
    with env(**c["envs"]):
        ch = gpu_lib.Chain(48000, C).add_fir(h, selector=sel, latency=c["latency"], block_hint=c["hint"])
        probe = ch.describe()[0]
        ch.close()
    B0, Bl, Rl = probe["levels"][0]["B"], probe["levels"][-1]["B"], probe["levels"][-1]["P"] + probe["bulk"] - 1
    # every ring wraps (FDL rows, V slots of the deepest tier), in whole calls
    nblk = max(2 * Rl + 3, 4 * max(probe["t_batch"], probe["t_far"]) + 3) * (Bl // B0) + 8 * (c["latency"] // B0 + 1)
    N = -(-nblk * B0 // c["call"]) * c["call"]
    x = dyadic_signal(rng, N, C)
    run = Runner(gpu_lib, c, x, h)
    base, plan, _ = run.run(device)
    again, plan2, dt = run.run(device)
    assert c["check"](plan), (case, plan)
    assert plan2 == plan, (case, plan, plan2)
    want = exact_conv(x, h, H_SHIFT, selector=sel, latency=c["latency"])
    r, m = fir_nerr(base, want, x, h, selector=sel)
    assert r <= FIR_RMS and m <= FIR_MAX, (case, mode, r, m, plan)
    d = _first_diff(again, base, B0)
    assert d is None, (case, mode, "two unstalled runs differ", d)
    block_us = 1e6 * dt / (N // B0)
    failures = []
    for roles, period, phase, times in _patterns(plan, device):
        us = int(min(max(times * block_us, STALL_MIN_US), STALL_MAX_US))
        gpu_lib.profile_read("fir_stall")
        gpu_lib.profile_enable(True)
        try:
            with stalled(gpu_lib, roles, us, period, phase):
                got, p, _ = run.run(device)
        finally:
            gpu_lib.profile_enable(False)
        ms, n_stalls = gpu_lib.profile_read("fir_stall")
        what = dict(case=case, mode=mode, role=ROLE_NAMES[roles], period=period, phase=phase, us=us)
        assert n_stalls > 0 and ms >= 0.9e-3 * us * n_stalls, (what, "the pattern delayed nothing", n_stalls, ms)
        assert p == plan, (what, p, plan)
        d = _first_diff(got, base, B0)
        if d is not None:
            failures.append(dict(what, **d))
    assert not failures, "\n".join(str(f) for f in failures)


def test_submit_wait_under_main_stream_stalls(gpu_lib):
    """Blocks in flight (submit_raw / wait, more than DONE_RING = 8 tickets outstanding) through eq -> fir_p -> resample
    on two slabs while the FIR delays each slab's stream (then also its side stream) by 2 ms on every block: bit-identical
    blocks and frame counts to synchronous calls of an unstalled chain."""
    from oracle import restate
    fs, C = 44100, 12
    h = restate.bench_ir(5000)
    coefs = eq_coefs(gpu_lib, fs, 3)
    rng = np.random.default_rng(7)
    sizes = [1024, 1024, 700, 1024, 1, 2048, 1024, 1024, 333] + [1024] * 15
    xs = [dyadic_signal(rng, n, C) for n in sizes]

    def make():
        return gpu_lib.Chain(fs, C, slabs_per_device=2).add_biquad(coefs).add_fir(h, block_hint=1024).add_resample(48000)

    a = make()
    want = [a.run(x).copy() for x in xs]
    out_max = a.max_out_frames(2048)
    a.close()
    ins = [gpu_lib.PinnedArray((2048, C)) for _ in xs]
    outs = [gpu_lib.PinnedArray((out_max + 1, C)) for _ in xs]
    for roles in (MAIN, MAIN | SIDE):
        b = make()
        gpu_lib.profile_read("fir_stall")
        gpu_lib.profile_enable(True)
        try:
            with stalled(gpu_lib, roles, 2000):
                tickets = []
                for i, x in enumerate(xs):
                    ins[i].array[:len(x)] = x
                    outs[i].array[:] = np.nan
                    tickets.append(b.submit_raw(len(x), ins[i].ptr, outs[i].ptr))
                got = []
                for i, (n, t) in enumerate(tickets):
                    b.wait(t)
                    got.append(outs[i].array[:n].copy())
        finally:
            gpu_lib.profile_enable(False)
        ms, n_stalls = gpu_lib.profile_read("fir_stall")
        b.close()
        # (the 2048-frame call re-plans the FIR to 2048-frame blocks: about 16 blocks per slab)
        assert n_stalls >= 2 * 8 and ms >= 0.9 * 2.0 * n_stalls, (roles, n_stalls, ms)
        for i, (w, g) in enumerate(zip(want, got)):
            assert w.shape == g.shape, (roles, i, w.shape, g.shape)
            assert np.array_equal(w, g), (roles, i, int(np.argmax(np.any(w != g, axis=1))))
    for p in ins + outs:
        p.free()


def test_debug_stall_rejects_bad_settings(gpu_lib):
    for args in ((16, 100, 1, 0), (MAIN, -1, 1, 0), (MAIN, 5001, 1, 0), (MAIN, 100, 0, 0), (MAIN, 100, 4, 4), (MAIN, 100, 4, -1)):
        with pytest.raises(gpu_lib.DspB200Error):
            gpu_lib.debug_stall(*args)
    gpu_lib.debug_stall(0)
