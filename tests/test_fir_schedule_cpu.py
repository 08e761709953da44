"""CPU tier: the FIR plan policy, fir_schedule() in dsp_b200/csrc/fir_plan.h, compiled with g++ alone.

The header needs no CUDA, so every plan the GPU tests assert through describe() is checked here against the same
tables (accuracy.FIR_CASES, accuracy.FIR_EDGES), on an H100's 132 SMs.  The driver calls FirKnobs::from_env(), so the
DSP_B200_FIR_* knobs go through the library's own parser.  Also checked: the benchmark's FIR configurations field by
field, the fold threshold, the knob parsing rules and scripts/fir_bytes.py's copy of the policy.
"""
import ctypes
import importlib.util
import json
import os

import pytest

from accuracy import F2, F4, FIR_CASES, FIR_EDGES, env, header_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMS = 132   # H100 SXM

DRIVER = r"""
#include "fir_plan.h"
using namespace dspb200;
// the schedule's describe() fields and `fold` as one JSON object; returns its length
extern "C" int schedule_json(long taps, long hint, int n_sel, int sm_count, char *out, int cap)
{
	const FirSchedule s = fir_schedule({ taps, hint, n_sel, sm_count, true, true }, FirKnobs::from_env());
	const std::string j = "{" + fir_schedule_json(s) + ",\"fold\":" + (s.fold ? "1" : "0") + "}";
	snprintf(out, cap, "%s", j.c_str());
	return (int) j.size();
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return header_lib(tmp_path_factory.mktemp("fir_schedule"), "firschedule", DRIVER)


@pytest.fixture
def plan(lib):
    def run(taps, hint, n_sel, **knobs):
        buf = ctypes.create_string_buffer(4096)
        with env(**{"DSP_B200_FIR_" + k: v for k, v in knobs.items()}):
            n = lib.schedule_json(ctypes.c_long(taps), ctypes.c_long(hint), n_sel, SMS, buf, len(buf))
        assert 0 < n < len(buf)
        return json.loads(buf.value.decode())
    return run


@pytest.fixture(autouse=True)
def default_knobs():
    """Every DSP_B200_FIR_* knob of the caller's environment unset: the cases below give the ones they mean."""
    with env(**{k: None for k in os.environ if k.startswith("DSP_B200_FIR_")}):
        yield


def _knobs(envs):
    return {k[len("DSP_B200_FIR_"):]: v for k, v in envs.items()}


@pytest.mark.parametrize("case", list(FIR_CASES))
def test_fir_cases(plan, case):
    frames, taps, C, hint, envs, check = FIR_CASES[case]
    p = plan(taps, hint or frames, C, **_knobs(envs))   # no hint: planned for the first call
    assert check(p), (case, p)


@pytest.mark.parametrize("case", list(FIR_EDGES))
def test_fir_edges(plan, case):
    e = FIR_EDGES[case]
    n_sel = e["C"] if e["sel"] is None else sum(e["sel"])
    p = plan(e["taps"], e["hint"], n_sel, **_knobs(e["envs"]))
    for k, v in e["plan"].items():
        assert p[k] == v, (case, k, p[k], v, p)


# bench.py's FIR workloads: (taps, channels, block) and the schedule each must get (config 5's filter is shared)
BENCH = {
    "headline": ((131072, 256, F4), dict(levels=[(F4, 32)], t_batch=8, fold=1, lookahead=2, stagger=1, pass_m=4,
                                               class_width=4, parts=(9, 2, 5))),
    "H_2048": ((131072, 256, F2), dict(levels=[(F2, 64)], t_batch=8, fold=1, lookahead=2, stagger=1, pass_m=4,
                                             class_width=4, parts=(9, 2, 5))),
    "C3": ((131072, 64, F4), dict(levels=[(F4, 32)], t_batch=4, fold=0, lookahead=3, stagger=1, pass_m=0,
                                        class_width=1, parts=(2, 2, 2))),
    "C5_share": ((65536, 256, F4), dict(levels=[(F4, 16)], t_batch=4, fold=1, lookahead=2, stagger=0, pass_m=0,
                                             class_width=1, parts=(5, 2, 5))),
}


@pytest.mark.parametrize("name", list(BENCH))
def test_bench_configs(plan, name):
    (taps, C, F), want = BENCH[name]
    p = plan(taps, F, C)
    want = dict(want)
    assert [(L["B"], L["P"]) for L in p["levels"]] == want.pop("levels"), p
    assert (p["l0_parts"], p["l0_parts_min"], p["l0_parts_steady"]) == want.pop("parts"), p
    want.update(t_far=0, far_e=0, far_classes=1, merge=0, tail_pf=2, bulk=1, pipe=0, pipe_pf=0)
    assert {k: p[k] for k in want} == want, p


@pytest.mark.parametrize("F,C,fold", [(F4, 66, 0), (F4, 67, 1), (F2, 132, 0), (F2, 133, 1)])
def test_fold_threshold(plan, F, C, fold):
    """Folded once the fused kernel's CTAs outnumber half the SMs: 2 ceil(C / CPB) > 132, CPB = 1 at 4096 frames and 2
    at 2048; the full-wave plan (depth 8, look-ahead 2) comes with it."""
    p = plan(131072, F, C)
    assert (p["fold"], p["lookahead"], p["t_batch"]) == ((1, 2, 8) if fold else (0, 3, 4)), p


def test_knob_parsing(plan):
    assert plan(131072, F4, 256)["t_batch"] == 8
    assert plan(131072, F4, 256, T=5)["t_batch"] == 4            # anything but 6, 8, 12 is 4
    assert plan(131072, F4, 256, T=12)["t_batch"] == 12
    assert plan(131072, F2, 8)["t_far"] == 8
    assert plan(131072, F2, 8, T2=10)["t_far"] == 0              # not a far-tier depth
    assert plan(131072, F2, 8, T2=8, FAR_CLASSES=2)["far_classes"] == 2
    assert plan(131072, F2, 8, T2=8, FAR_CLASSES=3)["far_classes"] == 1   # 8 / 3 turns: one
    assert plan(131072, F4, 256, PASS=2)["pass_m"] == 2
    assert plan(131072, F4, 256, PASS=8)["pass_m"] == 0          # outside [0, T)
    p = plan(131072, F4, 256, STAGGER=0)
    assert (p["stagger"], p["pass_m"], p["class_width"]) == (0, 0, 1), p
    p = plan(131072, F4, 64, FOLD=1)
    assert (p["fold"], p["lookahead"], p["l0_parts"]) == (1, 3, 6), p
    assert plan(131072, F4, 256, FOLD=0)["fold"] == 0
    p = plan(131072, F4, 8, MERGE=1)
    assert (p["merge"], p["fold"]) == (1, 0), p
    assert plan(131072, F4, 8, NO_BATCH=1)["t_batch"] == 0
    assert plan(3 * 8192 + 1, 4 * 8192, 3, NO_BULK=1)["bulk"] == 1
    assert plan(131072, 1024, 8, SINGLE_MIN=1024)["levels"] == [{"B": 1024, "P": 128}]


@pytest.fixture(scope="module")
def fir_bytes():
    spec = importlib.util.spec_from_file_location("fir_bytes_for_schedule", os.path.join(ROOT, "scripts", "fir_bytes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("block,C,t,lookahead,pass_m,unfolded", [
    (F4, 256, 8, 2, 4, False),   # the headline
    (F4, 8, 8, 3, 0, True),      # depth 8 on a plan that does not fold (DSP_B200_FIR_T=8)
    (F2, 256, 8, 2, 4, False),   # 2048-frame blocks, full-wave
    (F2, 8, 4, 3, 0, True),      # 2048-frame blocks with a far tier
])
def test_fir_bytes_plan_from_args(plan, fir_bytes, block, C, t, lookahead, pass_m, unfolded):
    """scripts/fir_bytes.py restates the policy for its byte model: it must agree with the library on every key."""
    class A:
        taps = 131072
    A.block, A.t, A.lookahead, A.pass_m, A.unfolded = block, t, lookahead, pass_m, unfolded
    want = fir_bytes.plan_from_args(A)
    p = plan(131072, block, C, T=t)
    assert {k: p[k] for k in want} == want, p
