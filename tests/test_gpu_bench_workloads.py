"""GPU tier: bench.py's workloads at their own shapes and in its launch regime, against exact and extended-precision
truths.

The benchmark keeps only a checksum of each workload's last block, and its input repeats every 8 blocks, so a read one
period off (an FDL row or a V slot 8 blocks stale, on a plan with 8 tier classes) would leave its numbers unchanged.
Here every workload runs as bench.time_device runs it, but on data that changes every block:

  - the input is aperiodic dyadic noise, uploaded once; right before each call the caller's stream copies the block
    into rotating buffer i % 8 (the headline) or i % 4 (the configs), the pools bench.py rotates;
  - the calls go back to back through run_device into ONE output buffer of max_out_frames(F) + 8 rows, and after each
    call the same stream copies the rows the call returned into a history;
  - the host waits once, after join.

FIR taps are bench.make_irs' decaying-noise IRs rounded onto the exact grid (accuracy.dyadic_taps), so the FIR
workloads are checked against accuracy.exact_conv on every channel.  H, H_2048 (three fresh chains, as the benchmark
makes them) and C3 share one input and one truth; the host-call workload e2e reuses them too.  Each workload's plan is
asserted from describe() (the records of tests/test_fir_schedule_cpu.py), and its streams run at least 2 P + 3 blocks
past the filter's first block, so that every FDL row, V slot and tier class wraps.

bench.time_device itself runs the headline on the benchmark's own IRs and 8-block pool: its last block, the one the
checksum and --dump-outputs come from, is checked against the periodic stream it computed.

The results may depend neither on the number of hardware queues (a child process, bench_workloads_child.py, runs the
device workloads with CUDA_DEVICE_MAX_CONNECTIONS=32, as bench.py sets it, and must give the same plans, frame counts
and output bits call by call) nor on the measurement modes bench.py switches on in the middle of a live chain's stream
(debug_serialize and profile_enable).

Errors are appended to the DSP_B200_ACCURACY_LOG file as test_gpu_accuracy does.  Measured on an H100 80GB HBM3 (700 W
limit), worst normalized RMS / max: H 4.9e-16 / 3.1e-15, H_2048 5.3e-16 / 3.5e-15, C3 4.8e-16 / 2.7e-15, e2e 4.8e-16 /
3.1e-15, time_device's last block 5.8e-16 (RMS relative to the stream); C5_share 1.8e-14 / 1.0e-13 relative to rms(want)
(bound 1e-12); C2 at most 0.012 of biquad_within_ref's bound; C4 1.4e-15 / 9.1e-15.  The whole file takes about 170 s
there, most of it the host truths.
"""
import hashlib
import json
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import bench
from accuracy import (biquad_truth, biquad_within_ref, bq_expect_launch, dyadic_signal, dyadic_taps, exact_conv, fir_nerr, nerr,
                      resample_truth, rs_counts)
from test_gpu_accuracy import FIR_MAX, FIR_RMS, H_SHIFT, _check_plan, _check_stream, _record, _tiled
from test_gpu_headline import FIR_TOL
from test_gpu_parity import BQ_TOL

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
DRIVER = os.path.join(HERE, "bench_workloads_child.py")
F4, F2 = 4096, 2048
FS, FS44 = bench.FS, 44100
C_H = bench.CHANNELS_PER_GPU
RS_BW = 0.939
FIR_BLOCKS = 75      # of 4096 frames: H (2 P + 3 + 8 = 75), C3 (>= 67), e2e; H_2048 runs the same input in 150 blocks (>= 139)

# describe() of each FIR workload (test_fir_schedule_cpu.BENCH)
_WAVE = dict(t_batch=8, t_far=0, stagger=1, class_width=4, lookahead=2, pass_m=4, tail_pf=2, l0_parts=9, l0_parts_min=2,
             l0_parts_steady=5)
FIR_PLANS = {
    "H": dict(_WAVE, levels=[{"B": F4, "P": 32}]),
    "H_2048": dict(_WAVE, levels=[{"B": F2, "P": 64}]),
    "C3": dict(levels=[{"B": F4, "P": 32}], t_batch=4, t_far=0, stagger=1, class_width=1, lookahead=3, pass_m=0, tail_pf=2,
               l0_parts=2, l0_parts_min=2, l0_parts_steady=2),
    "C5_share": dict(levels=[{"B": F4, "P": 16}], t_batch=4, t_far=0, stagger=0, class_width=1, lookahead=2, pass_m=0, tail_pf=2,
                     l0_parts=5, l0_parts_min=2, l0_parts_steady=5),
}
# name: (channels, block frames, blocks, rotating input buffers)
SHAPES = {"H": (C_H, F4, FIR_BLOCKS, 8), "H_2048": (C_H, F2, 2 * FIR_BLOCKS, 4), "C3": (64, F4, FIR_BLOCKS, 4),
          "C5_share": (C_H, F4, 35, 4), "C2": (C_H, F4, 40, 4), "C4": (1024, F4, 40, 4)}
CHILD_WORKLOADS = ["H", "H_2048", "C3", "C5_share", "C2", "C4"]

_cache = {}      # inputs and truths, shared by the tests of this module (cleared after it)
_records = {}    # name -> per-call record of the in-process run with the suite's own environment


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    _cache.clear()
    _records.clear()


def _cached(key, make):
    if key not in _cache:
        _cache[key] = make()
    return _cache[key]


# ------------------------------------------------------------------------------------------------------------
# inputs, chains and the launch regime
# ------------------------------------------------------------------------------------------------------------
def fir_input():
    """(x [75 * 4096, 256] dyadic noise, h [131072, 256]: bench.make_irs on the exact grid)."""
    def make():
        rng = np.random.default_rng(zlib.crc32(b"bench_workloads/fir"))
        return dyadic_signal(rng, FIR_BLOCKS * F4, C_H), dyadic_taps(bench.make_irs(bench.TAPS, C_H), H_SHIFT)
    return _cached("fir_input", make)


def fir_truth():
    """exact_conv of fir_input() in slabs of 32 channels (all 256 filter spectra at once would take 1 GB)."""
    def make():
        x, h = fir_input()
        return np.concatenate([exact_conv(x[:, a:a + 32], h[:, a:a + 32], H_SHIFT) for a in range(0, C_H, 32)], axis=1)
    return _cached("fir_truth", make)


def bases(name, k):
    """[frames, k] distinct dyadic noise signals, tiled over the channels of C5_share (4) and C4 (5)."""
    C, F, nblk, _ = SHAPES[name]
    return _cached("bases/" + name, lambda: dyadic_signal(np.random.default_rng(zlib.crc32(name.encode())), nblk * F, k))


def workload_input(name):
    """The whole input stream [blocks * F, C] of a device workload."""
    C, F, nblk, _ = SHAPES[name]
    if name in ("H", "H_2048", "C3"):
        return fir_input()[0][:, :C]
    if name == "C2":
        return _cached("x/C2", lambda: dyadic_signal(np.random.default_rng(zlib.crc32(b"C2")), nblk * F, C))
    return _tiled(bases(name, 4 if name == "C5_share" else 5), C)


def c5_taps():
    return dyadic_taps(bench.make_ir(65536, 0), H_SHIFT)


def make_chain(dsp, name, slabs=1):
    """The chain bench.py builds for a workload (measure_configs; the headline in main()), on the taps above."""
    C = SHAPES[name][0]
    if name in ("H", "H_2048", "C3"):
        return dsp.Chain(FS, C, devices=[0], slabs_per_device=slabs).add_fir(fir_input()[1][:, :C], block_hint=SHAPES[name][1])
    if name == "C2":
        return dsp.Chain(FS, C, devices=[0]).add_biquad(bench.eq_coefs(dsp, FS, 10))
    if name == "C4":
        return dsp.Chain(FS44, C, devices=[0]).add_resample(48000)
    return dsp.Chain(FS44, C, devices=[0]).add_biquad(bench.eq_coefs(dsp, FS44, 8)).add_fir(c5_taps(), block_hint=F4).add_resample(48000)


def device_stream(chain, x, F, pool, between=None):
    """bench.time_device's launch regime on data that changes every block (module docstring).  `between(i)`, when given,
    runs before block i is issued.  -> (history [frames out, C], per-call frame counts, per-call describe())."""
    import torch
    nblk, C = x.shape[0] // F, x.shape[1]
    stream = torch.cuda.current_stream().cuda_stream        # what bench.py issues on
    src = torch.from_numpy(np.ascontiguousarray(x[:nblk * F])).cuda()
    bufs = [torch.empty((F, C), dtype=torch.float64, device="cuda") for _ in range(pool)]
    of = chain.max_out_frames(F)
    d_out = torch.empty((of + 8, C), dtype=torch.float64, device="cuda")
    hist = torch.empty((nblk * of, C), dtype=torch.float64, device="cuda")
    counts, plans, pos = [], [], 0
    for i in range(nblk):
        if between:
            between(i)
        buf = bufs[i % pool]
        buf.copy_(src[i * F:(i + 1) * F])
        n = chain.run_device(0, F, buf.data_ptr(), d_out.data_ptr(), stream)
        hist[pos:pos + n].copy_(d_out[:n])
        counts.append(n)
        plans.append(chain.describe())
        pos += n
    chain.join(0, stream)
    torch.cuda.synchronize()
    out = hist[:pos].cpu().numpy()
    del src, bufs, d_out, hist
    return out, counts, plans


def record(hist, counts, plans):
    """Per call: describe() after it, its frame count and the SHA-256 of its output rows."""
    rows = np.split(hist, np.cumsum(counts)[:-1])
    return [dict(plan=p, frames=int(n), sha256=hashlib.sha256(np.ascontiguousarray(r).tobytes()).hexdigest())
            for p, n, r in zip(plans, counts, rows)]


def run_workload(dsp, name):
    """One fresh chain of the workload through device_stream; -> (history, counts, plans)."""
    C, F, nblk, pool = SHAPES[name]
    ch = make_chain(dsp, name)
    try:
        return device_stream(ch, workload_input(name), F, pool)
    finally:
        ch.close()


def record_of(dsp, name):
    """The per-call record of a workload, from the in-process run when a test has made it."""
    if name not in _records:
        _records[name] = record(*run_workload(dsp, name))
    return _records[name]


def _host_stream(dsp, name, x):
    """The same chain in host mode (run(), the library's own buffers and streams), block by block."""
    F = SHAPES[name][1]
    ch = make_chain(dsp, name)
    try:
        outs = [ch.run(x[i:i + F]).copy() for i in range(0, x.shape[0], F)]
    finally:
        ch.close()
    return np.concatenate(outs), [o.shape[0] for o in outs]


def _op(plans, op):
    return [p for p in plans if p["op"] == op][0]


def _fir_check(name, got, C):
    x, h = fir_input()
    n = got.shape[0]
    r, m = fir_nerr(got, fir_truth()[:n, :C], x[:n, :C], h[:, :C])
    _record("fir", "bench/" + name, rms=r, max=m)
    assert r <= FIR_RMS and m <= FIR_MAX, (name, r, m)


# ------------------------------------------------------------------------------------------------------------
# the FIR workloads
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["H", "C3"])
def test_fir_workload_exact(gpu_lib, name):
    """H (256 channels x 131072 taps, 4096-frame blocks: the folded, staggered full-wave plan with the mid-window pass;
    256 fused-kernel CTAs on 132 SMs, so the tier CTAs queue between its waves) and C3 (64 channels: the per-block MAC
    form) in the benchmark's launch regime, every channel against the exact convolution."""
    C, F, nblk, pool = SHAPES[name]
    hist, counts, plans = run_workload(gpu_lib, name)
    _records[name] = record(hist, counts, plans)
    _check_plan(_op(plans[-1], "fir"), FIR_PLANS[name], name)
    assert counts == [F] * nblk
    _fir_check(name, hist, C)


def test_fir_workload_2048_three_fresh_chains(gpu_lib):
    """H_2048 (256 channels, 2048-frame blocks: 64 partitions, the same tier shape) on three fresh chains, as the
    benchmark measures it: the three bit-identical, and against the exact convolution on every channel."""
    C, F, nblk, pool = SHAPES["H_2048"]
    runs = [run_workload(gpu_lib, "H_2048") for _ in range(3)]
    hist, counts, plans = runs[0]
    _records["H_2048"] = record(hist, counts, plans)
    _check_plan(_op(plans[-1], "fir"), FIR_PLANS["H_2048"], "H_2048")
    assert counts == [F] * nblk
    for k, (other, _, _) in enumerate(runs[1:]):
        assert np.array_equal(other, hist), "fresh chain %d differs from the first" % (k + 2)
    del runs
    _fir_check("H_2048", hist, C)


def test_e2e_host_calls_sync_and_in_flight(gpu_lib):
    """e2e: H's filter and input through run_host on 4 channel slabs, from pinned buffers (inputs write-combined, 8 of
    them refilled in turn, one output buffer), then through submit/wait with 3 blocks in flight on a fresh chain (4
    output buffers): both against H's exact truth, and bit-identical to each other.  Each slab plans its 64 channels
    as C3 does (per-block MAC, look-ahead 3)."""
    x, _ = fir_input()
    C, F, nblk, depth = C_H, F4, FIR_BLOCKS, 3
    pins = [gpu_lib.PinnedArray((F, C), write_combined=True) for _ in range(8)]
    pouts = [gpu_lib.PinnedArray((F, C)) for _ in range(depth + 1)]
    sync, piped = np.empty((nblk * F, C)), np.empty((nblk * F, C))
    try:
        ch = make_chain(gpu_lib, "H", slabs=4)
        assert ch.n_shards == 4
        for i in range(nblk):
            pins[i % 8].array[:] = x[i * F:(i + 1) * F]
            assert ch.run_raw(F, pins[i % 8].ptr, pouts[0].ptr) == F
            sync[i * F:(i + 1) * F] = pouts[0].array
        ch.close()
        ch = make_chain(gpu_lib, "H", slabs=4)
        tickets = []
        for i in range(nblk + depth):
            if i < nblk:
                pins[i % 8].array[:] = x[i * F:(i + 1) * F]      # its last user, block i - 8, was waited for at i - 5
                n, t = ch.submit_raw(F, pins[i % 8].ptr, pouts[i % (depth + 1)].ptr)
                assert n == F
                tickets.append(t)
            if i >= depth:
                j = i - depth
                ch.wait(tickets[j])
                piped[j * F:(j + 1) * F] = pouts[j % (depth + 1)].array
        plan = ch.describe()[0]
        ch.close()
    finally:
        for p in pins + pouts:
            p.free()
    _check_plan(plan, dict(FIR_PLANS["C3"], n_sel=C // 4), "e2e")    # a slab of 64 channels plans as C3 does
    _fir_check("e2e", sync, C)
    assert np.array_equal(piped, sync), "submit/wait differs from the synchronous calls"


def test_bench_time_device_last_block(gpu_lib):
    """bench.time_device itself on a fresh headline chain with the benchmark's IRs and 8-block pool (warm-up 8, 67
    timed steps): the block it leaves in d_out -- what the checksum and --dump-outputs report -- against the periodic
    stream it computed, over the last P + 2 blocks (enough for 131072 taps), at the headline's tolerance."""
    import torch
    from oracle import restate
    C, F, warm, steps = C_H, F4, 8, 67
    irs = bench.make_irs(bench.TAPS, C)
    blocks = [bench.make_block(F, C, i) for i in range(8)]
    ch = gpu_lib.Chain(FS, C, devices=[0]).add_fir(irs, block_hint=F)
    try:
        d_blocks = [torch.from_numpy(b).cuda() for b in blocks]
        d_out = torch.empty((F, C), dtype=torch.float64, device="cuda")
        bench.time_device(ch, d_blocks, d_out.data_ptr(), F, steps, warm, torch.cuda.current_stream().cuda_stream)
        got = d_out.cpu().numpy()
        plan = ch.describe()[0]
    finally:
        ch.close()
    _check_plan(plan, FIR_PLANS["H"], "time_device")
    P = plan["levels"][0]["P"]
    order = [i % 8 for i in range(warm)] + [i % 8 for i in range(steps)]    # the blocks time_device issued
    tail = np.concatenate([blocks[k] for k in order[-(P + 2):]])
    want = restate.fir_stream(tail, irs)[-F:]
    r = nerr(got, want)[0]
    _record("fir", "bench/time_device_last_block", rms=r)
    assert r <= FIR_TOL, r


# ------------------------------------------------------------------------------------------------------------
# the configs with biquads and the resampler
# ------------------------------------------------------------------------------------------------------------
def test_c5_share_chain(gpu_lib):
    """C5_share: 8 eq + a shared 65536-tap FIR (folded, unstaggered, look-ahead 2, 16 partitions) + resample 44100 ->
    48000 on 256 channels, 4 distinct signals tiled over them: per-call counts as rs_counts replays them, the copies bit
    for bit, and the 4 bases against the composed truth (long-double cascade, FIR, long-double resampler) within
    test_gpu_parity's chain bound, on the first and last 200 outputs and a seeded sample of the others."""
    C, F, nblk, pool = SHAPES["C5_share"]
    hist, counts, plans = run_workload(gpu_lib, "C5_share")
    _records["C5_share"] = record(hist, counts, plans)
    _check_plan(_op(plans[-1], "fir"), FIR_PLANS["C5_share"], "C5_share")
    assert counts == rs_counts(FS44, 48000, [F] * nblk, bw=RS_BW)[0]
    assert np.array_equal(hist, _tiled(hist[:, :4], C)), "channels with the same input differ"
    from oracle import restate
    base = bases("C5_share", 4)
    y = restate.fir_stream(biquad_truth(base, bench.eq_coefs(gpu_lib, FS44, 8)).astype(np.float64), c5_taps())
    n = hist.shape[0]
    rng = np.random.default_rng(5)
    rows = np.unique(np.concatenate([np.arange(200), np.arange(n - 200, n), rng.choice(n, 3600, replace=False)]))
    want = resample_truth(y, FS44, 48000, RS_BW, n, rows=rows).astype(np.float64)
    r, m = nerr(hist[rows, :4], want)
    _record("chain", "bench/C5_share", rms=r, max=m)
    assert r <= BQ_TOL, (r, m)


def test_c2_eq_cascade(gpu_lib):
    """C2: 10 eq stages on 256 channels (two channels per CTA): bit-identical to the host-mode stream of the same chain,
    and biquad_within_ref on both channels of the first CTA, two in the middle and both of the last CTA."""
    C, F, nblk, pool = SHAPES["C2"]
    hist, counts, plans = run_workload(gpu_lib, "C2")
    _records["C2"] = record(hist, counts, plans)
    x = workload_input("C2")
    coefs = bench.eq_coefs(gpu_lib, FS, 10)
    bq, want = _op(plans[-1], "biquad"), bq_expect_launch(C, 10, F)
    assert (bq["ch"], bq["split"]) == (want["ch"], want["split"]) == (2, 0), bq
    assert counts == [F] * nblk
    host, _ = _host_stream(gpu_lib, "C2", x)
    assert np.array_equal(hist, host), "device-resident calls differ from host mode"
    cols = [0, 1, 126, 127, 254, 255]
    errs = biquad_within_ref(hist[:, cols], x[:, cols], coefs)
    _record("biquad", "bench/C2", err_gpu=max(e[0] for e in errs), ratio=max(e[2] for e in errs))


def test_c4_resample(gpu_lib):
    """C4: 44100 -> 48000 on 1024 channels (the tensor-core kernel), 5 distinct signals tiled over them: per-call
    counts as rs_counts replays them, bit-identical to the host-mode stream, the copies bit for bit and the bases within
    test_gpu_accuracy's resampler bounds."""
    C, F, nblk, pool = SHAPES["C4"]
    hist, counts, plans = run_workload(gpu_lib, "C4")
    _records["C4"] = record(hist, counts, plans)
    assert _op(plans[-1], "resample")["kernel"] == "k_rs_mma2", plans[-1]
    assert counts == rs_counts(FS44, 48000, [F] * nblk, bw=RS_BW)[0]
    host, hcounts = _host_stream(gpu_lib, "C4", workload_input("C4"))
    assert hcounts == counts
    assert np.array_equal(hist, host), "device-resident calls differ from host mode"
    del host
    _check_stream("bench/C4", hist, bases("C4", 5), FS44, 48000, RS_BW)


# ------------------------------------------------------------------------------------------------------------
# independence from the hardware queues and from the measurement modes
# ------------------------------------------------------------------------------------------------------------
def test_measurement_modes_mid_stream(gpu_lib):
    """What bench.py does to the headline chain after its timed loop: join and synchronise after block 24, switch
    debug_serialize and profile_enable on for 16 blocks (everything on the caller's stream, event brackets around the
    kernels), synchronise, switch both off and finish the stream.  Every call bit-identical to the uninterrupted one."""
    import torch
    C, F, nblk, pool = SHAPES["H"]
    want = record_of(gpu_lib, "H")
    ch = make_chain(gpu_lib, "H")
    stream = torch.cuda.current_stream().cuda_stream
    k = 24

    def between(i):
        if i == k:
            ch.join(0, stream)
            torch.cuda.synchronize()
            gpu_lib.debug_serialize(True)
            gpu_lib.profile_enable(True)
        elif i == k + 16:
            torch.cuda.synchronize()
            gpu_lib.profile_enable(False)
            gpu_lib.debug_serialize(False)
    try:
        got = record(*device_stream(ch, workload_input("H"), F, pool, between))
    finally:
        gpu_lib.profile_enable(False)
        gpu_lib.debug_serialize(False)
        ch.close()
    profiled = {name: gpu_lib.profile_read(name)[1] for name in ("fir_level0", "fir_mac", "fir_mac_batch", "fir_mac_batch_far")}
    assert profiled["fir_level0"] == 16, profiled       # the fused kernel of each block while profiling was on
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, ("call %d differs" % i, k)
    assert len(got) == len(want) == nblk


def test_results_do_not_depend_on_connection_count(gpu_lib, tmp_path):
    """A child process started with CUDA_DEVICE_MAX_CONNECTIONS=32 in its environment (set before CUDA starts, as
    bench.py sets it; the suite runs with the driver's default) runs H, H_2048, C3, C5_share, C2 and C4 on the same
    inputs: every call's plan, frame count and output bits equal this process's.  The paths carry no atomics, so the
    output may not depend on how the streams are scheduled."""
    import torch
    mine = {name: record_of(gpu_lib, name) for name in CHILD_WORKLOADS}
    torch.cuda.empty_cache()
    out = tmp_path / "child.json"
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    p = subprocess.run([sys.executable, DRIVER, str(out)], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, "child failed (rc %d):\n%s" % (p.returncode, p.stderr[-6000:])
    child = json.loads(out.read_text())
    assert child["CUDA_DEVICE_MAX_CONNECTIONS"] == "32", child["CUDA_DEVICE_MAX_CONNECTIONS"]
    assert sorted(child["workloads"]) == sorted(CHILD_WORKLOADS)
    here = os.environ.get("CUDA_DEVICE_MAX_CONNECTIONS")
    for name in CHILD_WORKLOADS:
        theirs = child["workloads"][name]
        assert len(theirs) == len(mine[name]), name
        for i, (a, b) in enumerate(zip(mine[name], theirs)):
            assert a == b, (name, "call %d" % i, "connections here: %s" % here)
