"""CPU tier: scripts/fir_bytes.py's byte model of the full-wave FIR plan (near tier of depth 8, look-ahead 2; DESIGN.md K2)."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fb():
    spec = importlib.util.spec_from_file_location("fir_bytes_for_full_wave", os.path.join(ROOT, "scripts", "fir_bytes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def plan(B, P, t, la, t_far=0):
    """A folded single-level plan as describe() reports it."""
    return {"levels": [{"B": B, "P": P}], "tail_pf": 2, "t_batch": t, "t_far": t_far, "far_e": t if t_far else 0,
            "stagger": 0 if t_far else 1, "merge": 0, "pipe": 0, "pipe_pf": 0, "l0_parts": t + la - 1, "l0_parts_min": la,
            "lookahead": la}


def test_headline_full_wave(fb):
    total, parts = fb.folded_bytes_model(plan(4096, 32, 8, 2), 1)
    # fused kernel: 2 .. 9 partitions, 5.5 on average, 4.5 FDL rows: 8 + 16 + 72 + 88 + 16 + 24 = 224
    # near tier: 30 FDL rows + 30 filter rows + 8 V rows per launch of 8 periods = 136
    assert parts["fir_level0"] == 224 and parts["fir_mac_batch"] == 136 and "fir_mac" not in parts
    assert total == 360


def test_headline_depth8_lookahead3(fb):
    total, parts = fb.folded_bytes_model(plan(4096, 32, 8, 3), 1)
    assert parts["fir_level0"] == 256 and parts["fir_mac_batch"] == 132 and total == 388


def test_lookahead_absent_is_3(fb):
    p = plan(4096, 32, 4, 3)
    del p["lookahead"]
    assert fb.folded_bytes_model(p, 1)[0] == fb.folded_bytes_model(plan(4096, 32, 4, 3), 1)[0] == 440


def test_near_tier_reads_p_minus_la_rows(fb):
    # per launch: P - la FDL rows, P - la filter rows (none with a shared IR), T rows of V
    for B, P, t, la in ((4096, 32, 8, 2), (4096, 19, 8, 2), (4096, 18, 4, 2), (2048, 64, 8, 2), (4096, 32, 4, 3)):
        for h in (0, 1):
            _, parts = fb.folded_bytes_model(plan(B, P, t, la), h)
            assert parts["fir_mac_batch"] == 16.0 * ((P - la) * (1 + h) + t) / t, (B, P, t, la, h)


def test_plan_from_args_lookahead(fb):
    class A:
        taps, block, t, unfolded, lookahead = 131072, 4096, 8, False, 2
    p = fb.plan_from_args(A)
    assert (p["l0_parts"], p["l0_parts_min"], p["lookahead"]) == (9, 2, 2) and fb.folded_bytes_model(p, 1)[0] == 360
    A.lookahead = 3
    assert fb.folded_bytes_model(fb.plan_from_args(A), 1)[0] == 388
