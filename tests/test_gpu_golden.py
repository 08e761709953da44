"""GPU tier: every committed golden vector (outputs of the reference's own code, see
tests/golden/make_golden.py) through the CUDA path, called via the C ABI.  Tolerance from the
north star: <= 1e-6 RMS in double; the kernels are held to 1e-13 of the golden output's RMS here."""
import os

import numpy as np
import pytest

from accuracy import nerr
from conftest import rms

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TOL = 1e-13   # rms(got - want) / rms(want)
BQ_TOL = 1e-12   # the biquad vector's low-corner eq: the FP64 reference's own rounding is ~3e-13 of it

NAMES = ["gain", "biquad", "fir_p", "fir_p_2ch", "fir", "fir_direct", "hilbert", "resample_up", "resample_down",
         "resample_2x", "chain"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: z[k] for k in z.files}


@pytest.mark.parametrize("name", NAMES)
def test_golden(gpu_lib, name):
    from dsp_b200.effects import build_chain
    g = load(name)
    ec = build_chain(str(g["chain"]), int(g["fs"]), int(g["channels"]), dir=GOLDEN)
    y, counts = ec.process(g["x"], int(g["block"]))
    assert ec.fs_out == int(g["out_fs"])
    assert y.shape == g["y"].shape, (y.shape, g["y"].shape)
    assert list(counts) == list(g["counts"])
    assert nerr(y, g["y"])[0] <= (BQ_TOL if name == "biquad" else TOL), rms(y - g["y"])
    assert np.max(np.abs(y - g["y"])) <= 1e-9
    ec.close()


@pytest.mark.parametrize("name", ["biquad", "fir_p", "hilbert", "resample_up", "chain"])
@pytest.mark.parametrize("block", [1, 7, 64, 1000])
def test_golden_streaming_invariance(gpu_lib, name, block):
    """Same stream cut into different call sizes gives the same stream (state carry-over)."""
    from dsp_b200.effects import build_chain
    g = load(name)
    x = g["x"][:600] if block == 1 else g["x"]
    ec = build_chain(str(g["chain"]), int(g["fs"]), int(g["channels"]), dir=GOLDEN)
    y, _ = ec.process(x, block)
    n = min(y.shape[0], g["y"].shape[0], int(x.shape[0] * ec.fs_out / int(g["fs"])) - 400 if "resample" in name or name == "chain" else x.shape[0])
    assert n > 100
    assert nerr(y[:n], g["y"][:n])[0] <= (BQ_TOL if name == "biquad" else TOL)
    ec.close()


@pytest.mark.parametrize("name", ["biquad", "fir_p_2ch", "chain"])
def test_golden_sharded_equals_single(gpu_lib, name):
    """Channel slabs are independent: a chain cut into shards is bit-identical to one shard."""
    from dsp_b200.effects import build_chain
    g = load(name)
    a = build_chain(str(g["chain"]), int(g["fs"]), int(g["channels"]), dir=GOLDEN)
    b = build_chain(str(g["chain"]), int(g["fs"]), int(g["channels"]), dir=GOLDEN, slabs_per_device=2)
    assert b.chain.n_shards == 2
    ya, ca = a.process(g["x"], int(g["block"]))
    yb, cb = b.process(g["x"], int(g["block"]))
    assert ca == cb
    assert np.array_equal(ya, yb)
    a.close()
    b.close()


def test_reset_restores_initial_state(gpu_lib):
    from dsp_b200.effects import build_chain
    g = load("chain")
    ec = build_chain(str(g["chain"]), int(g["fs"]), int(g["channels"]), dir=GOLDEN)
    y1 = np.concatenate([ec.run(g["x"][i:i + 512]) for i in range(0, 2048, 512)])
    ec.reset()
    y2 = np.concatenate([ec.run(g["x"][i:i + 512]) for i in range(0, 2048, 512)])
    assert np.array_equal(y1, y2)
    ec.close()
