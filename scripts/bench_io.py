"""Host-call cost of the sample formats at the I/O edge (the _io entry points, edge.cu).

    python scripts/bench_io.py [--steps 400] [--warmup 16] [--repeats 3] [--out FILE]

Two workloads of 256 channels in 4096-frame blocks on 4 channel slabs: the headline chain (fir_p, 131072 taps per
channel) and a link-bound chain (gain only).  Each runs in three formats, the same one in and out: f64 interleaved (the
plain ABI), f32 interleaved and f32 planar ([channels, frames]), through the synchronous host call and through
submit/wait with 3 blocks in flight, on page-locked buffers.  The formats alternate within each of `repeats` rounds;
the result is the median over rounds and its spread (max - min).  Then the edge kernels alone: k_edge_in + k_edge_out
timed with CUDA events around each launch (the library's "edge" profile) on 4096- and 65536-frame blocks, as bytes
per second against the data sheet's 3.35 TB/s of an H100 SXM -- the kernels' share of peak, not the call's.  The card's
name and power limit are read in the same run and printed with the figures.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dsp_b200  # noqa: E402
from dsp_b200 import IO_F32, IO_F64, IO_PLANAR  # noqa: E402

FS, C, F, SLABS, DEPTH, TAPS = 48000, 256, 4096, 4, 3, 131072
HBM_PEAK = 3.35e12
FORMATS = {"f64_interleaved": IO_F64, "f32_interleaved": IO_F32, "f32_planar": IO_F32 | IO_PLANAR}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown (nvidia-smi: %s)" % r.stdout.strip()


class Pinned:
    """A page-locked host array of `dtype` (dspb200_host_alloc)."""

    def __init__(self, shape, dtype, write_combined=False):
        dtype = np.dtype(dtype)
        n = int(np.prod(shape))
        alloc = dsp_b200.lib().dspb200_host_alloc_wc if write_combined else dsp_b200.lib().dspb200_host_alloc
        self.ptr = alloc(n * dtype.itemsize)
        if not self.ptr:
            raise RuntimeError("host_alloc: " + dsp_b200.last_error())
        buf = (ctypes.c_char * (n * dtype.itemsize)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=dtype, count=n).reshape(shape)

    def free(self):
        self.array = None
        dsp_b200.lib().dspb200_host_free(self.ptr)


def make_chain(workload):
    ch = dsp_b200.Chain(FS, C, slabs_per_device=SLABS)
    if workload == "headline":
        rng = np.random.default_rng(7)
        h = rng.standard_normal((TAPS, C)) * np.exp(-np.arange(TAPS) / 20000.0)[:, None] * 0.01
        ch.add_fir(h, block_hint=F)
    else:
        ch.add_gain(0.5)
    return ch


def run_format(ch, fmt, blocks_in, outs, steps, warmup):
    """(synchronous ms per block, submit/wait ms per block) of `steps` blocks after `warmup`."""
    stride = F if fmt & IO_PLANAR else 0
    n_in = len(blocks_in)
    for i in range(warmup):
        ch.run_io_raw(F, blocks_in[i % n_in].ptr, fmt, stride, outs[0].ptr, fmt, stride)
    t0 = time.perf_counter()
    for i in range(steps):
        ch.run_io_raw(F, blocks_in[i % n_in].ptr, fmt, stride, outs[0].ptr, fmt, stride)
    ch.sync()
    sync_ms = (time.perf_counter() - t0) / steps * 1e3
    tickets = []
    t0 = time.perf_counter()
    for i in range(steps):
        _, t = ch.submit_io_raw(F, blocks_in[i % n_in].ptr, fmt, stride, outs[i % (DEPTH + 1)].ptr, fmt, stride)
        tickets.append(t)
        if i >= DEPTH:
            ch.wait(tickets[i - DEPTH])
    for t in tickets[-DEPTH:]:
        ch.wait(t)
    pipe_ms = (time.perf_counter() - t0) / steps * 1e3
    return sync_ms, pipe_ms


def edge_alone(frames, reps):
    """k_edge_in + k_edge_out on one 256-channel block of `frames` frames (f32 in and out, an empty chain, Mode D):
    microseconds per launch and bytes/s per layout, from CUDA events around each launch."""
    import torch
    res = {}
    ch = dsp_b200.Chain(FS, C)
    for name, fmt in (("f32_interleaved", IO_F32), ("f32_planar", IO_F32 | IO_PLANAR)):
        x = torch.randn(C * frames, dtype=torch.float32, device="cuda")
        y = torch.empty_like(x)
        stride = frames if fmt & IO_PLANAR else 0
        for _ in range(3):
            ch.run_device_io(0, frames, x.data_ptr(), fmt, stride, y.data_ptr(), fmt, stride, None)
        torch.cuda.synchronize()
        dsp_b200.profile_read("edge")
        dsp_b200.profile_enable(True)
        for _ in range(reps):
            ch.run_device_io(0, frames, x.data_ptr(), fmt, stride, y.data_ptr(), fmt, stride, None)
        torch.cuda.synchronize()
        ms, n = dsp_b200.profile_read("edge")
        dsp_b200.profile_enable(False)
        assert torch.equal(x, y), "the edge round trip f32 -> f64 -> f32 must be exact"
        us = ms / n * 1e3
        byts = C * frames * (4 + 8)   # each kernel reads one format and writes the other
        res[name] = {"us_per_kernel": us, "bytes_per_kernel": byts, "GBs": byts / (us * 1e-6) / 1e9,
                     "share_of_hbm_peak": byts / (us * 1e-6) / HBM_PEAK, "launches_timed": n}
    ch.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if dsp_b200.device_count() < 1:
        raise SystemExit("bench_io: no CUDA device (nothing here runs on the CPU)")
    import torch
    torch.cuda.init()
    out = {"card": card(), "channels": C, "frames_per_block": F, "channel_slabs": SLABS, "blocks_in_flight": DEPTH,
           "steps": a.steps, "warmup": a.warmup, "repeats": a.repeats, "workloads": {}}
    rng = np.random.default_rng(1)
    base = [(rng.standard_normal((F, C)) * 0.2).astype(np.float32) for _ in range(4)]
    for workload in ("gain", "headline"):
        ch = make_chain(workload)
        bufs = {}
        for name, fmt in FORMATS.items():
            dt = np.float32 if fmt & IO_F32 else np.float64
            shape = (C, F) if fmt & IO_PLANAR else (F, C)
            ins = [Pinned(shape, dt, write_combined=True) for _ in base]
            for p, b in zip(ins, base):
                p.array[:] = b.T if fmt & IO_PLANAR else b
            bufs[name] = (fmt, ins, [Pinned(shape, dt) for _ in range(DEPTH + 1)])
        rounds = {name: [] for name in FORMATS}
        for r in range(a.repeats):
            for name, (fmt, ins, outs) in bufs.items():
                rounds[name].append(run_format(ch, fmt, ins, outs, a.steps, a.warmup))
        w = {}
        for name, rs in rounds.items():
            sync, pipe = [x[0] for x in rs], [x[1] for x in rs]
            esize = 4 if FORMATS[name] & IO_F32 else 8
            w[name] = {"sync_us_per_block": statistics.median(sync) * 1e3, "sync_spread_us": (max(sync) - min(sync)) * 1e3,
                       "submit_us_per_block": statistics.median(pipe) * 1e3, "submit_spread_us": (max(pipe) - min(pipe)) * 1e3,
                       "link_bytes_per_block_each_way": C * F * esize,
                       "sync_Msamples_s": C * F / statistics.median(sync) / 1e3,
                       "submit_Msamples_s": C * F / statistics.median(pipe) / 1e3}
        # the outputs of the three formats agree (f32 outputs are the f64 ones rounded)
        ref = bufs["f64_interleaved"][2][0].array.astype(np.float32)
        for name in ("f32_interleaved", "f32_planar"):
            got = bufs[name][2][0].array
            got = got.T if FORMATS[name] & IO_PLANAR else got
            w[name]["same_as_f64_rounded"] = bool(np.array_equal(got, ref))
        out["workloads"][workload] = w
        ch.close()
        for _, ins, outs in bufs.values():
            for p in ins + outs:
                p.free()
    out["edge_kernels"] = {"frames_%d" % fr: edge_alone(fr, reps) for fr, reps in ((4096, 400), (65536, 50))}
    out["card_after"] = card()
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
