"""GPU tier: composed device chains against the same operators run one chain at a time.

Every operator is deterministic, so a chain of several operators must give bit-identical output, with identical
per-call frame counts, to a pipeline of one-operator chains (same devices, slabs, block hints, selectors and taps),
each call's output fed to the next chain as one call.  That pins the routing of `Shard::run_ops` (which of the shard's
buffers each operator reads and writes, in place or not), where a rate-changing operator's output goes, how the drain
feeds the operators after the draining one, and when the shard buffers grow -- with no tolerance to tune.

Chains (every one also with a 20000-frame call in the middle of the stream, which grows the shard buffers):
  A  44.1 kHz: gain (mult + add), 20 per-channel biquad stages (two operators: 16 + 4), resample 48000, per-channel
     20000-tap FIR with one channel passed through, 3 biquad stages at 48 kHz, align with delays and a discard;
  B  48 kHz: resample 96000, fir.c's FFT path (latency = its length), biquad, resample 44100, gain;
  C  48 kHz: biquad, the full-wave FIR plan (18 * 4096 + 1 taps in 4096-frame blocks, channels from the SM count), gain.
Layouts: A and B at 7 channels in 1 and 3 slabs (2 + 2 + 3) and 12 in 3; C in one slab (full-wave) and in two.
Call modes: run_host with ragged calls and a reset mid-stream, submit/wait with up to 12 blocks in flight (the 8-slot
completion ring waits internally) and one synchronous call among them, run_device out of place per shard on the
torch stream, and (C) in place; after each one the drain, then reset, the stream again and a drain that stays dry
(the resampler's drain counters survive a reset).  Chain A is also checked against the float64 composition of the
restated references, so that a fault shared by the one-operator and the composed paths cannot hide.
The whole file takes about 35 s (measured on an H100 80GB HBM3 at its 700 W limit).
"""
import functools
import zlib

import numpy as np
import pytest

from accuracy import nerr
from test_gpu_accuracy import bq_check
from test_gpu_fir_full_wave import full_wave_channels

pytestmark = pytest.mark.gpu

F = 4096
# ragged calls: single frames, one short of / exactly / one past a block, three blocks and a bit, a short call, a
# 20000-frame call that grows the shard buffers mid-stream, and 367 frames that bring the stream back to a multiple of
# 4096 so that the whole-block calls after it are aligned (the FIR's fused and full-wave paths)
HEAD = [1, 7, F - 1, F, F + 1, 3 * F + 5, 100, 20000, 367]
WHOLE = {"A": 8, "B": 8, "C": 12}          # 4096-frame calls after the ragged head
POLLS = [1, 7, F]                          # drain poll sizes; the last one repeats until the drain is dry
DEPTH = 12                                 # blocks in flight in the submit mode (the completion ring holds 8)
RUN_AT, SWAP_AT = 14, 4                    # submit mode: the synchronous call, and where a newer ticket is waited first
ALIGN_DELAYS = [0, 1, 700, 5000, 3, 0, 64, 4097, 2, 0, 333, 1]
# layouts whose slabs do not all run the same kernels agree to the tolerance of the operator whose kernel differs:
# the resampler (test_gpu_parity.TOL) in A and B, the FIR plan (test_gpu_parity.FIR_TOL) in C
LAYOUT_TOL = {"A": 1e-13, "B": 1e-13, "C": 1e-14}
BQ_TOL = 1e-12                             # test_gpu_parity.test_full_size_config5_chain_share


# ------------------------------------------------------------------------------------------------------------
# the chains: every per-channel parameter depends on the channel index alone, so a chain on fewer channels is the
# leading channels of a chain on more
# ------------------------------------------------------------------------------------------------------------
def _eq(gpu_lib, fs, sections):
    return np.array([gpu_lib.biquad_design(13, fs, f, q, g) for f, q, g in sections])


def _spec_a(gpu_lib, C):
    from oracle import restate
    k = np.arange(C)
    bq = np.zeros((20, C, 5))
    for s in range(20):
        for c in range(C):
            bq[s, c] = gpu_lib.biquad_design(13, 44100, 40.0 * 1.3 ** s + 3 * c, 0.7 + 0.1 * (c % 5), ((5 * s + 3 * c) % 13 - 6) * 0.5)
    sel = [c != 5 for c in range(C)]
    h = np.stack([restate.bench_ir(20000, c) for c in range(C) if sel[c]], axis=1)
    return 44100, [
        ("gain", dict(mult=0.5 + 0.05 * k, add=0.01 * (k - 3))),
        ("biquad", dict(coefs=bq)),
        ("resample", dict(out_fs=48000)),
        ("fir", dict(taps=h, selector=sel, block_hint=F)),
        ("biquad", dict(coefs=_eq(gpu_lib, 48000, [(120.0, 1.0, 3.0), (2500.0, 0.8, -4.0), (11000.0, 1.2, 2.0)]))),
        ("align", dict(delay=[ALIGN_DELAYS[c % len(ALIGN_DELAYS)] for c in range(C)], discard_frames=1000)),
    ]


def _spec_b(gpu_lib, C):
    from oracle import restate
    taps = 2000
    return 48000, [
        ("resample", dict(out_fs=96000)),
        ("fir", dict(taps=restate.bench_ir(taps), latency=restate.next_fast_fftw_len(taps))),
        ("biquad", dict(coefs=_eq(gpu_lib, 96000, [(60.0, 0.9, 4.0), (15000.0, 1.5, -3.0)]))),
        ("resample", dict(out_fs=44100)),
        ("gain", dict(mult=1.5 - 0.1 * np.arange(C))),
    ]


def _spec_c(gpu_lib, C):
    from oracle import restate
    h = np.stack([restate.bench_ir(18 * F + 1, c) for c in range(C)], axis=1)
    return 48000, [
        ("biquad", dict(coefs=_eq(gpu_lib, 48000, [(80.0, 0.7, 5.0), (6000.0, 1.1, -2.5)]))),
        ("fir", dict(taps=h, block_hint=F)),
        ("gain", dict(mult=0.25 + 0.01 * np.arange(C))),
    ]


SPECS = {"A": _spec_a, "B": _spec_b, "C": _spec_c}


@functools.lru_cache(maxsize=None)
def _spec(gpu_lib, name, C):
    return SPECS[name](gpu_lib, C)


@functools.lru_cache(maxsize=None)
def _inputs(name, C):
    sizes = HEAD + [F] * WHOLE[name]
    x = np.stack([np.random.default_rng(zlib.crc32(b"chain%d" % c)).standard_normal(sum(sizes)) for c in range(C)], axis=1) * 0.2
    return tuple(np.split(x, np.cumsum(sizes)[:-1]))


def _add_ops(ch, ops):
    for kind, kw in ops:
        getattr(ch, "add_" + kind)(**kw)
    return ch


def _op_index(ops, gpu_ops_per_op):
    """Index of each FIR among the chain's device operators (a biquad of more than 16 stages is several)."""
    pos = np.cumsum([0] + list(gpu_ops_per_op))
    return [int(pos[i]) for i, (kind, _) in enumerate(ops) if kind == "fir"]


class Pipeline:
    """The oracle: one Chain per operator at the rate that operator sees, each call's output fed to the next chain as
    one call.  A call that yields no frames stops there (run_ops skips operators on 0 frames).  The drain is replayed
    as drain_host does it: each chain in order is polled with the poll size carried through the earlier chains'
    max_out_frames, up to the first that is not dry, whose output runs through the chains after it."""

    def __init__(self, gpu_lib, fs, C, slabs, ops):
        self.chains = []
        for op in ops:
            ch = _add_ops(gpu_lib.Chain(fs, C, slabs_per_device=slabs), [op])
            self.chains.append(ch)
            fs = ch.out_fs
        self.fir = [i for i, (kind, _) in enumerate(ops) if kind == "fir"]

    @staticmethod
    def _through(y, chains):
        for ch in chains:
            if y.shape[0] == 0:
                break
            y = ch.run(y).copy()
        return y

    def run(self, x):
        return self._through(x, self.chains)

    def drain(self, frames):
        for i, ch in enumerate(self.chains):
            y = ch.drain(frames)
            if y is not None:
                return self._through(y, self.chains[i + 1:])
            frames = ch.max_out_frames(frames)
        return None

    def reset(self):
        for ch in self.chains:
            ch.reset()

    def paths(self):
        return [self.chains[i].describe()[0]["paths"] for i in self.fir]

    def close(self):
        for ch in self.chains:
            ch.close()


def _drain_all(ch):
    """Poll at 1, 7, 4096, 4096, ... frames; the polls' outputs, ending with None (dry)."""
    outs = []
    for i in range(64):
        y = ch.drain(POLLS[min(i, len(POLLS) - 1)])
        outs.append(y)
        if y is None:
            return outs
    raise AssertionError("the drain did not run dry in 64 polls")


def _same(got, want, what):
    """Bit-identical call by call: the same frame counts, the same doubles (None: a dry drain poll)."""
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        if g is None or w is None:
            assert g is None and w is None, (what, i, "dry on one side only")
            continue
        assert g.shape == w.shape, (what, i, g.shape, w.shape)
        if not np.array_equal(g, w):
            d = np.abs(g - w)
            bad = np.argwhere(d > 0)
            raise AssertionError("%s: call %d differs in %d samples, first at (frame, channel) %s, max |diff| %.3g"
                                 % (what, i, len(bad), tuple(bad[0]), float(d.max())))


@functools.lru_cache(maxsize=None)
def _reference(gpu_lib, name, C, slabs):
    """The pipeline's record of the stream, its FIR paths, the drain, and after reset the stream and a dry drain."""
    fs, ops = _spec(gpu_lib, name, C)
    xs = _inputs(name, C)
    pipe = Pipeline(gpu_lib, fs, C, slabs, ops)
    try:
        stream = [pipe.run(x) for x in xs]
        paths = pipe.paths()
        drain = _drain_all(pipe)
        pipe.reset()
        again = [pipe.run(x) for x in xs]
        dry = _drain_all(pipe)
        n_ops = [ch.n_ops for ch in pipe.chains]
    finally:
        pipe.close()
    _same(again, stream, "pipeline after reset")
    assert dry == [None], "pipeline: the drain after a reset is not dry"
    if any(kind == "resample" for kind, _ in ops):
        assert len(drain) > 2 and sum(y.shape[0] for y in drain[:-1]) > 0, "pipeline: nothing drained"
    return dict(stream=stream, paths=paths, drain=drain, dry=dry, n_ops=n_ops)


# ------------------------------------------------------------------------------------------------------------
# the composed chain in each call mode
# ------------------------------------------------------------------------------------------------------------
def _run_host(ch, xs):
    return [ch.run(x).copy() for x in xs]


def _run_submit(gpu_lib, ch, xs):
    """submit_raw / wait with up to DEPTH blocks in flight on pinned buffers; call RUN_AT is a synchronous run()
    between two submits, and at SWAP_AT the second-oldest ticket is waited for before the oldest."""
    C = ch.channels
    ins = [gpu_lib.PinnedArray(x.shape) for x in xs]
    outs = [gpu_lib.PinnedArray((max(ch.max_out_frames(x.shape[0]), 1), C)) for x in xs]
    got, pending = [None] * len(xs), []

    def collect(j, m, t):
        ch.wait(t)
        got[j] = outs[j].array[:m].copy()
    try:
        for i, x in enumerate(xs):
            if i == RUN_AT:
                got[i] = ch.run(x).copy()
                continue
            ins[i].array[...] = x
            n, t = ch.submit_raw(x.shape[0], ins[i].ptr, outs[i].ptr)
            pending.append((i, n, t))
            if i == SWAP_AT:
                a, b = pending.pop(0), pending.pop(0)
                collect(*b)
                collect(*a)
            while len(pending) > DEPTH:
                collect(*pending.pop(0))
        for p in pending:
            collect(*p)
    finally:
        ch.sync()
        for p in ins + outs:
            p.free()
    return got


def _run_device(ch, xs, in_place=False):
    """run_device per shard on the torch stream: each shard's channels sliced into a buffer of their own."""
    import torch
    st = torch.cuda.current_stream().cuda_stream
    shards = [ch.shard_info(s) for s in range(ch.n_shards)]
    calls, keep = [], []
    for x in xs:
        f = x.shape[0]
        parts, counts = [], set()
        for s, (_, b, n) in enumerate(shards):
            d_in = torch.from_numpy(np.ascontiguousarray(x[:, b:b + n])).cuda()
            d_out = d_in if in_place else torch.empty((max(ch.max_out_frames(f), 1), n), dtype=torch.float64, device="cuda")
            counts.add(ch.run_device(s, f, d_in.data_ptr(), d_out.data_ptr(), st))
            parts.append(d_out)
            keep.append(d_in)
        assert len(counts) == 1, ("shards disagree on the frame count", counts)
        calls.append((counts.pop(), parts))
    # nothing orders the torch stream against the shard streams the drain and the host calls use
    torch.cuda.synchronize()
    return [np.concatenate([p[:m].cpu().numpy() for p in parts], axis=1) for m, parts in calls]


CASES = [("A", 7, 1), ("A", 7, 3), ("A", 12, 3), ("B", 7, 1), ("B", 7, 3), ("B", 12, 3), ("C", None, 1), ("C", None, 2)]
MODES = ["host", "submit", "device"]
PARAMS = [(n, C, s, m) for n, C, s in CASES for m in MODES + (["device_in_place"] if n == "C" else [])]


@pytest.mark.parametrize("name,C,slabs,mode", PARAMS, ids=["%s-%sch-%dslab-%s" % (n, C or "fw", s, m) for n, C, s, m in PARAMS])
def test_composed_chain_equals_operator_pipeline(gpu_lib, name, C, slabs, mode):
    """The stream, every FIR's paths, the drain, and after reset the stream and a dry drain, bit for bit against the
    pipeline of one-operator chains; the host mode also resets mid-stream and must replay a fresh chain's output."""
    C = C or full_wave_channels(F)
    fs, ops = _spec(gpu_lib, name, C)
    ref = _reference(gpu_lib, name, C, slabs)
    xs = _inputs(name, C)
    ch = _add_ops(gpu_lib.Chain(fs, C, slabs_per_device=slabs), ops)
    try:
        assert ch.n_shards == slabs and ch.n_ops == sum(ref["n_ops"]), (ch.n_shards, ch.n_ops, ref["n_ops"])
        if name == "A":
            assert ref["n_ops"][1] == 2   # 20 biquad stages: operators of 16 + 4
        fir_at = _op_index(ops, ref["n_ops"])
        if name == "C":
            plan = ch.describe()[fir_at[0]]
            assert plan["levels"] == [{"B": F, "P": 19}] and plan["tail_pf"] == 2, plan
            if slabs == 1:
                assert (plan["lookahead"], plan["t_batch"]) == (2, 8), ("not the full-wave plan", plan)
            else:
                assert plan["lookahead"] == 3, ("half the channels per slab must not be full-wave", plan)
        if mode == "host":
            got = _run_host(ch, xs)
        elif mode == "submit":
            got = _run_submit(gpu_lib, ch, xs)
        else:
            got = _run_device(ch, xs, in_place=(mode == "device_in_place"))
        _same(got, ref["stream"], mode)
        desc = ch.describe()
        assert [desc[i]["paths"] for i in fir_at] == ref["paths"], ([desc[i]["paths"] for i in fir_at], ref["paths"])
        if mode == "host":
            ch.reset()
            _same(_run_host(ch, xs), ref["stream"], "host, after a reset mid-stream")
        _same(_drain_all(ch), ref["drain"], mode + ", drain")
        ch.reset()
        _same(_run_host(ch, xs), ref["stream"], mode + ", after the drain and a reset")
        _same(_drain_all(ch), ref["dry"], mode + ", drain after a reset")
    finally:
        ch.close()


@pytest.mark.parametrize("name", ["A", "B", "C"])
def test_layouts_agree(gpu_lib, name):
    """Different slab layouts of one chain.  Bit for bit where every slab runs the same kernels: the first 4-channel
    slab of 12 channels in 3 slabs against 4 channels in one slab (A, B).  Otherwise to the tolerance of the operator
    whose kernel differs, with identical frame counts: 7 channels in 1 slab against 3 slabs and against the leading
    channels of 12 in 3 (the resampler runs single channels on 7 and 3 channels, channel pairs on 2 and the tensor
    cores on 4), and C in one slab (full-wave FIR plan) against two (per-block MAC plan)."""
    def whole(r):
        return r["stream"] + [y for y in r["drain"] if y is not None]

    def close(a, b, n_ch, what):
        ga, gb = whole(a), whole(b)
        assert [y.shape[0] for y in ga] == [y.shape[0] for y in gb], what
        ya, yb = np.concatenate(ga)[:, :n_ch], np.concatenate(gb)[:, :n_ch]
        for c in range(n_ch):
            e = nerr(ya[:, c], yb[:, c])[0]
            assert e <= LAYOUT_TOL[name], (what, c, e)

    if name == "C":
        C = full_wave_channels(F)
        close(_reference(gpu_lib, "C", C, 1), _reference(gpu_lib, "C", C, 2), C, "1 slab vs 2")
        return
    r71, r73 = _reference(gpu_lib, name, 7, 1), _reference(gpu_lib, name, 7, 3)
    r123, r41 = _reference(gpu_lib, name, 12, 3), _reference(gpu_lib, name, 4, 1)
    close(r71, r73, 7, "7 channels: 1 slab vs 3")
    close(r71, r123, 7, "7 channels in 1 slab vs 12 in 3")
    _same([y[:, :4] for y in r123["stream"]], r41["stream"], "12 in 3 slabs, first slab vs 4 channels in 1 slab")
    _same([None if y is None else y[:, :4] for y in r123["drain"]], r41["drain"], "drain, first slab vs 4 channels")


def test_chain_a_matches_float64_composition(gpu_lib):
    """The composed chain A (7 channels, one slab) against the float64 composition of the restated references over the
    first six calls: gain, restate.biquad_cascade, restate.Resampler, restate.fir_stream, restate.biquad_cascade and
    the align's delays and discard applied in numpy; RMS error per channel <= 1e-12 of rms(want)."""
    from oracle import restate
    C, n_calls = 7, 6
    fs, ops = _spec(gpu_lib, "A", C)
    xs = _inputs("A", C)[:n_calls]
    ch = _add_ops(gpu_lib.Chain(fs, C), ops)
    got = np.concatenate(_run_host(ch, xs))
    ch.close()
    kw = [k for _, k in ops]
    y = np.concatenate(xs) * kw[0]["mult"] + kw[0]["add"]
    y = restate.biquad_cascade(y, kw[1]["coefs"])
    y = restate.Resampler(fs, kw[2]["out_fs"], C).run(y)
    y = restate.fir_stream(y, kw[3]["taps"], selector=kw[3]["selector"])
    y = restate.biquad_cascade(y, kw[4]["coefs"])
    want = np.zeros_like(y)
    for c, d in enumerate(kw[5]["delay"]):
        want[d:, c] = y[:y.shape[0] - d, c]
    want = want[kw[5]["discard_frames"]:]
    m = min(got.shape[0], want.shape[0])
    assert m > 20000, (got.shape, want.shape)
    for c in range(C):
        e = nerr(got[:m, c], want[:m, c])[0]
        assert e <= BQ_TOL, (c, e)


@pytest.mark.parametrize("stages,n_ops", [(15, 1), (16, 2)])
def test_absorb_fuses_biquads_up_to_16_stages(gpu_lib, stages, n_ops):
    """Absorbing a 1-stage chain into a 15-stage chain fuses the two into one operator; into a 16-stage chain it does
    not (16 stages per operator at most).  Either way the cascade is within bq_check of the long-double truth."""
    fs, C = 48000, 3
    rng = np.random.default_rng(stages)
    coefs = np.array([[gpu_lib.biquad_design(13, fs, 50.0 * 1.25 ** s + 7 * c, 0.8 + 0.1 * c, rng.uniform(-5, 5))
                       for c in range(C)] for s in range(stages + 1)])
    a = gpu_lib.Chain(fs, C).add_biquad(coefs[:stages])
    b = gpu_lib.Chain(fs, C).add_biquad(coefs[stages:])
    a.absorb(b)
    assert (a.n_ops, b.n_ops) == (n_ops, 0)
    x = rng.standard_normal((3 * F + 11, C)) * 0.2
    got = np.concatenate([a.run(x[i:i + 1000]).copy() for i in range(0, x.shape[0], 1000)])
    a.close()
    b.close()
    bq_check("absorb_%d+1" % stages, got, x, coefs)


# ------------------------------------------------------------------------------------------------------------
# in-place device calls on a chain whose last operator changes the frame count
# ------------------------------------------------------------------------------------------------------------
def _in_place_chain(gpu_lib, case, fs, C):
    ch = gpu_lib.Chain(fs, C)
    if case == "biquad_resample":
        return ch.add_biquad(_eq(gpu_lib, fs, [(200.0, 0.9, 6.0), (3000.0, 1.3, -3.0)])).add_resample(48000)
    if case == "gain_align":
        return ch.add_gain([0.5, -1.0, 2.0, 0.25]).add_align([0, 3, 700, 1], 500)
    return ch.add_align([0, 3, 700, 1], 500).add_biquad(_eq(gpu_lib, fs, [(200.0, 0.9, 6.0)]))


def _device_stream(ch, x, n, in_place=False):
    import torch
    st = torch.cuda.current_stream().cuda_stream
    calls = []
    for i in range(0, x.shape[0], n):
        d_in = torch.from_numpy(np.ascontiguousarray(x[i:i + n])).cuda()
        f = d_in.shape[0]
        d_out = d_in if in_place else torch.empty((max(ch.max_out_frames(f), 1), x.shape[1]), dtype=torch.float64, device="cuda")
        calls.append((ch.run_device(0, f, d_in.data_ptr(), d_out.data_ptr(), st), d_out, d_in))
    torch.cuda.synchronize()
    return [d_out[:m].cpu().numpy() for m, d_out, _ in calls]


@pytest.mark.parametrize("case", ["biquad_resample", "gain_align"])
def test_run_device_in_place_rejected_without_side_effects(gpu_lib, case):
    """run_device(d, d) on a chain whose last operator changes the frame count is an error, and it has no effect: the
    buffer keeps its bytes, and the out-of-place calls that follow give the stream of a chain that never saw it."""
    import torch
    fs, C, n = 44100, 4, 1024
    x = np.random.default_rng(zlib.crc32(case.encode())).standard_normal((5 * n + 3, C)) * 0.2
    a, b = _in_place_chain(gpu_lib, case, fs, C), _in_place_chain(gpu_lib, case, fs, C)
    st = torch.cuda.current_stream().cuda_stream
    d = torch.from_numpy(x[:n].copy()).cuda()
    before = d.clone()
    with pytest.raises(gpu_lib.DspB200Error, match="in-place"):
        a.run_device(0, n, d.data_ptr(), d.data_ptr(), st)
    torch.cuda.synchronize()
    assert torch.equal(d.view(torch.int64), before.view(torch.int64)), "the rejected call changed the caller's buffer"
    _same(_device_stream(a, x, n), _device_stream(b, x, n), case + ": after the rejected call vs a fresh chain")
    a.close()
    b.close()


def test_run_device_in_place_before_a_frame_count_change(gpu_lib):
    """In place stays allowed when the operator that changes the frame count is not the last one ([align, biquad]:
    align writes to a scratch buffer): the same stream as out of place."""
    fs, C, n = 44100, 4, 1024
    x = np.random.default_rng(3).standard_normal((5 * n + 3, C)) * 0.2
    a, b = _in_place_chain(gpu_lib, "align_biquad", fs, C), _in_place_chain(gpu_lib, "align_biquad", fs, C)
    got = _device_stream(a, x, n, in_place=True)
    _same(got, _device_stream(b, x, n), "align, biquad: in place vs out of place")
    assert sum(y.shape[0] for y in got) == x.shape[0] - 500
    a.close()
    b.close()
