"""CPU tier: scripts/fir_bytes.py's byte model of the mid-window pass of the full-wave FIR plan (DESIGN.md K2)."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fb():
    spec = importlib.util.spec_from_file_location("fir_bytes_for_pass", os.path.join(ROOT, "scripts", "fir_bytes.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def plan(t, m, la=2, B=4096, P=32):
    """A staggered folded single-level plan with one tier and a pass of depth m (0: none), as describe() reports it."""
    return {"levels": [{"B": B, "P": P}], "tail_pf": 2, "t_batch": t, "t_far": 0, "far_e": 0, "stagger": 1, "merge": 0,
            "pipe": 0, "pipe_pf": 0, "l0_parts": t + la - 1, "l0_parts_min": la, "lookahead": la, "pass_m": m,
            "l0_parts_steady": la - 1 + max(m, t - m) if m else t + la - 1}


@pytest.mark.parametrize("t,m,fused,tier,pas,total", [
    (8, 0, 224, 136, None, 360),
    (8, 2, 176, 136, 42, 354),
    (8, 4, 160, 136, 38, 334),
    (8, 6, 176, 136, 34, 346),
    (12, 6, 192, 96, 16.0 * 29 / 12, 48 + 144 + 96 + 16.0 * 29 / 12),
])
def test_headline_pass_table(fb, t, m, fused, tier, pas, total):
    # fused kernel 48 + 32 lp: lp = 2 + (m(m-1)/2 + (T-m)(T-m-1)/2) / T; pass: m + (T-1) + 2 (T-m) rows per T blocks
    got, parts = fb.folded_bytes_model(plan(t, m), 1)
    assert parts["fir_level0"] == pytest.approx(fused) and parts["fir_mac_batch"] == pytest.approx(tier), parts
    assert parts.get("fir_mac_batch_pass") == (None if pas is None else pytest.approx(pas)), parts
    assert got == pytest.approx(total)


def test_default_and_deep_totals(fb):
    assert fb.folded_bytes_model(plan(8, 4), 1)[0] == 334
    assert round(fb.folded_bytes_model(plan(12, 6), 1)[0], 2) == 326.67
    assert fb.folded_bytes_model(plan(8, 0), 1)[0] == 360


def test_shared_ir_pass_reads_no_filter_rows(fb):
    _, parts = fb.folded_bytes_model(plan(8, 4), 0)
    assert parts["fir_mac_batch_pass"] == 16.0 * (4 + 2 * 4) / 8


def test_plan_from_args_pass(fb):
    class A:
        taps, block, t, unfolded, lookahead, pass_m = 131072, 4096, 8, False, 2, 4
    p = fb.plan_from_args(A)
    assert (p["pass_m"], p["l0_parts"], p["l0_parts_steady"], p["l0_parts_min"]) == (4, 9, 5, 2)
    assert fb.folded_bytes_model(p, 1)[0] == 334
    A.lookahead = 3   # the pass is for look-ahead 2 only
    p = fb.plan_from_args(A)
    assert p["pass_m"] == 0 and fb.folded_bytes_model(p, 1)[0] == 388
    A.lookahead, A.pass_m = 2, 0
    assert fb.folded_bytes_model(fb.plan_from_args(A), 1)[0] == 360
