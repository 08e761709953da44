"""CPU tier: scripts/fir_bytes.py's byte model of the folded FIR tail with the near tier's triangle (DESIGN.md K2)."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fb():
    spec = importlib.util.spec_from_file_location("fir_bytes_for_model", os.path.join(ROOT, "scripts", "fir_bytes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def plan(B, P, t=4, t_far=0, lp_min=3, **kw):
    p = {"levels": [{"B": B, "P": P}], "tail_pf": 2, "t_batch": t, "t_far": t_far, "far_e": t if t_far else 0,
         "stagger": 0 if t_far else 1, "merge": 0, "pipe": 0, "pipe_pf": 0, "l0_parts": t + 2, "l0_parts_min": lp_min}
    p.update(kw)
    return p


def test_headline_triangle(fb):
    total, parts = fb.folded_bytes_model(plan(4096, 32), 1)
    # fused kernel: (3 + 6) / 2 = 4.5 partitions on average, 3.5 FDL rows: 8 + 16 + 56 + 72 + 16 + 24 = 192
    # near tier: 236 as before + H_3 .. H_5 once per 4 periods = 248
    assert parts["fir_level0"] == 192 and parts["fir_mac_batch"] == 248 and "fir_mac" not in parts
    assert total == 440


def test_headline_rectangle_as_before(fb):
    total, parts = fb.folded_bytes_model(plan(4096, 32, lp_min=6), 1)
    assert parts["fir_level0"] == 240 and parts["fir_mac_batch"] == 236 and total == 476


def test_2048_blocks_two_tiers(fb):
    total, parts = fb.folded_bytes_model(plan(2048, 64, t_far=8), 1)
    assert parts["fir_level0"] == 192 and parts["fir_mac_batch"] == 120 and parts["fir_mac_batch_far"] == 230
    assert total == 542


def test_shared_ir_saves_fdl_rows_only(fb):
    tri, _ = fb.folded_bytes_model(plan(4096, 32), 0)
    rect, _ = fb.folded_bytes_model(plan(4096, 32, lp_min=6), 0)
    assert rect - tri == 24


def test_plan_from_args_matches_the_library_plan(fb):
    class A:
        taps, block, t, unfolded = 131072, 4096, 4, False
    p = fb.plan_from_args(A)
    assert (p["l0_parts"], p["l0_parts_min"]) == (6, 3) and fb.folded_bytes_model(p, 1)[0] == 440
    A.t = 8
    assert fb.folded_bytes_model(fb.plan_from_args(A), 1)[0] == 388
    A.t, A.unfolded = 4, True
    assert fb.folded_bytes_model(fb.plan_from_args(A), 1)[0] == 508
