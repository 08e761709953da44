"""CPU tier: the FIR tail schedule of dsp_b200/csrc/fir_plan.h, compiled with g++ alone.

For every plan with a tail (the pipeline kernel's aside) the whole-block schedule fir.cu runs is enumerated from the
header alone (fir_tail_steps(), fir_fused_read() and the functions they use): the fused kernel of every block (one stream,
in order), the per-block MAC or the merged grid (a side stream), the tier launches (a second side stream), over enough
blocks to pass start-up and wrap the V and FDL rings several times.  Then:

1. exactly once: every partition p <= j of every period j of every channel is summed by exactly one launch;
2. causality: a launch after block q reads only blocks <= q;
3. FDL reuse: a launch that reads block b is ordered before the fused kernel of block b + R, which overwrites its row;
4. V, V2 and Y slots: every write of a period is ordered before its readers, no write of another period of the slot
   lands in between, and every write is read (a reader that finds no write reads the zeros of an unwritten slot);
5. event rings: the event each wait uses still marks the block it means when the wait is enqueued.

"Ordered" follows from in-order streams, "ev_main and ev_urgent mark the fused kernel of their block" and "a wait on a
ring slot orders after the last record into it".  Each check is shown to fail on a broken copy of the headline's records.
"""
import copy
import ctypes
import os
from collections import defaultdict

import numpy as np
import pytest

from accuracy import F2, F4, FIR_CASES, FIR_EDGES, FOLD_CASES, PASS_CASES, env, header_lib

SMS = 132   # H100 SXM

DRIVER = r"""
#include "fir_plan.h"
using namespace dspb200;
static FirSchedule g;
static FirTailRing r;
extern "C" void plan(long taps, long hint, int n_sel, int sm_count, int *o)
{
	g = fir_schedule({ taps, hint, n_sel, sm_count, true, true }, FirKnobs::from_env());
	r = {};
	const FirLevelPlan &L = g.lv[g.n_levels - 1];
	const int v[] = { g.n_levels, L.P, L.R, g.tail_pf, g.t_batch, g.t_far, g.fold, g.stagger, g.merge_tail, g.use_pipe,
	                  g.mac_parts().first, g.mac_parts().second, g.v_slots(0), g.v_slots(1), g.y_slots() };
	for (int i = 0; i < 15; ++i) o[i] = v[i];
}
extern "C" FirTailSteps tail_steps(long q, int n_sel) { return fir_tail_steps(g, q, n_sel, r); }
extern "C" FirTailRead fused_read(long j) { return fir_fused_read(g, j, r); }
extern "C" const int consts[] = { FIR_N_EV_BS, FIR_N_BS_AT, FIR_N_EV_BATCH, FIR_N_EV_TAIL, sizeof(FirTailSteps), sizeof(FirTailRead) };
// as fir.cu's fused kernel gets it: K = T classes when staggered, else 1; at most l0_parts()
extern "C" int fused_parts(long blk, int s)
{
	return fir_fused_parts(blk, s, g.t_batch, g.stagger ? g.t_batch : 1, g.class_w, g.la, g.pass_m, g.l0_parts());
}
extern "C" FirBatchWindow batch_window(bool pass, int T, int p_lo, int p_hi, int pass_m) { return fir_batch_window(pass, T, p_lo, p_hi, pass_m); }
extern "C" int class_channel(int g_, int K, int w, int y) { return fir_class_channel(g_, K, w, y); }
"""
PLAN_KEYS = ("n_levels", "P", "R", "tail_pf", "t_batch", "t_far", "fold", "stagger", "merge", "pipe", "mac_lo", "mac_hi",
             "V_slots", "V2_slots", "Y_slots")
EV = (None, "ev_main", "ev_urgent", "ev_tail", "ev_batch", "ev_bs")   # FirEvRing
MAC, MERGED, TIER = range(3)                                          # FirTailKind
RINGS = {}   # the header's event rings, read when it is compiled (lib)


def _struct(*fields):   # the layout of one of fir_plan.h's structs
    return type("S", (ctypes.Structure,), dict(_fields_=[f if isinstance(f, tuple) else (f, ctypes.c_int) for f in fields]))


Ev = _struct("ring", "slot", ("blk", ctypes.c_long))
TierLaunch = _struct("tier", "T", "g", "K", "w", "pf", "p_lo", "p_hi", "rows", ("from_far", ctypes.c_bool), "pass_g", "pass_rows",
                     "pass_m")
TailStep = _struct("kind", "role", ("wait", Ev * 2), ("rec", Ev * 2), ("j", ctypes.c_long), "y", "v", ("d", TierLaunch))
TailSteps = _struct("n", ("l", TailStep * 3))
TailRead = _struct(("wait", Ev), "y", "v")
BatchWindow = _struct("x_hi", "h_hi", "n_t")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = header_lib(tmp_path_factory.mktemp("fir_tiers"), "firtiers", DRIVER)
    lib.tail_steps.argtypes, lib.tail_steps.restype = [ctypes.c_long, ctypes.c_int], TailSteps
    lib.fused_read.argtypes, lib.fused_read.restype = [ctypes.c_long], TailRead
    lib.fused_parts.argtypes = [ctypes.c_long, ctypes.c_int]
    lib.batch_window.argtypes, lib.batch_window.restype = [ctypes.c_bool] + [ctypes.c_int] * 4, BatchWindow
    o = list((ctypes.c_int * 6).in_dll(lib, "consts"))
    RINGS.update(zip(("ev_bs", "ev_bs_at", "ev_batch", "ev_tail"), o))
    assert o[4:] == [ctypes.sizeof(TailSteps), ctypes.sizeof(TailRead)]   # the header's layout
    return lib


def _plans():
    """id -> (taps, hint, channels, envs): FIR_CASES, FIR_EDGES, the benchmark's FIR configurations, the full-wave
    channel counts and the shapes of the fold and pass GPU tests in both their forms."""
    out = {}
    for name, (frames, taps, C, hint, envs, _) in FIR_CASES.items():
        out["case/" + name] = (taps, hint or frames, C, envs)
    for name, e in FIR_EDGES.items():
        out["edge/" + name] = (e["taps"], e["hint"], e["C"] if e["sel"] is None else sum(e["sel"]), e["envs"])
    for name, (taps, C, F) in (("headline", (131072, 256, F4)), ("H_2048", (131072, 256, F2)), ("C3", (131072, 64, F4)),
                               ("C5_share", (65536, 256, F4))):
        out["bench/" + name] = (taps, F, C, {})
    out["full_wave/72x4096"] = (131072, F4, 72, {})
    out["full_wave/136x2048"] = (131072, F2, 136, {})
    for name, (taps, B, P, envs, T, m) in PASS_CASES.items():
        for mm in (T // 2 if m is None else m, 0):
            out["pass/%s/m%d" % (name, mm)] = (taps, B, 72 if B == F4 else 136, dict(envs, DSP_B200_FIR_PASS=mm))
    for name, (taps, C, B, envs, _) in FOLD_CASES.items():
        for fold in (1, 0):
            out["fold/%s/%d" % (name, fold)] = (taps, B, C, dict(envs, DSP_B200_FIR_FOLD=fold))
    return out


PLANS = _plans()


class Schedule:
    """The whole-block schedule of one plan: launch records in issue order and the event operations between them."""

    def __init__(self, lib, taps, hint, C, envs):
        o = (ctypes.c_int * len(PLAN_KEYS))()
        with env(**{k: None for k in os.environ if k.startswith("DSP_B200_FIR_")}):
            with env(**envs):
                lib.plan(ctypes.c_long(taps), ctypes.c_long(hint), C, SMS, o)
        self.lib, self.C = lib, C
        self.p = dict(zip(PLAN_KEYS, o))
        p = self.p
        self.has_tail = p["tail_pf"] > 0 and not p["pipe"]
        self.P, self.R = p["P"], p["R"]
        self.Q = 3 * self.P + 4 * max(p["t_batch"], p["t_far"], 1) + 4
        self.slots = dict(V=p["V_slots"], V2=p["V2_slots"], Y=p["Y_slots"])

    def tier_parts(self, q, d, sums, reads, vacc):
        """Add the sums, reads and vacc of the tier launch d after block q (and of the mid-window pass it runs)."""
        for pass_, g, rows in ((False, d.g, d.rows), (True, d.pass_g, d.pass_rows)):
            if rows == 0:
                continue
            ch = np.array([self.lib.class_channel(g, d.K, d.w, y) for y in range(rows)], dtype=np.int64)
            w = self.lib.batch_window(pass_, d.T, d.p_lo, d.p_hi, d.pass_m)
            x_hi, h_hi, n_t = w.x_hi, w.h_hi, w.n_t
            pf = d.pf
            reads.append((q + pf + 1 - (x_hi - 1), q))   # FDL rows m in [pf+1, x_hi): X_{q+pf+1-m}
            for t in range(n_t):
                j = q + pf + 1 + t
                sums.append((ch, j, max(pf + 1 + t, d.p_lo), min(x_hi + t, h_hi)))
                if pass_:
                    vacc.append((ch, "V", j, "acc"))
                else:
                    vacc.append((ch, "V2" if d.tier else "V", j, "init"))
                    if d.from_far:
                        vacc.append((ch, "V2", j, "read"))

    def enumerate(self):
        """-> (records, ops).  A record is one launch: id, stream, kind, q (the block it follows; a fused kernel's own
        block), waits (ids it is ordered after), sums [(channels, period, first partition, end)], reads [(first block,
        last block)] of the FDL, vacc [(channels, buffer, period, "init" | "acc" | "read")].  ops: the host's event
        operations in issue order, ("rec" | "wait", ring, index, block or period it marks / must mark)."""
        p, lib, C = self.p, self.lib, self.C
        allc = np.arange(C)
        recs, ops = [], []
        marks = {}                    # (ring, slot) -> the record last recorded into it
        tier_upto = []                # tier_upto[q]: the last tier record issued after a block <= q

        def rec(stream, kind, q, waits, sums=(), reads=(), vacc=()):
            recs.append(dict(id=len(recs), stream=stream, kind=kind, q=q, waits=[w for w in waits if w is not None],
                             sums=list(sums), reads=list(reads), vacc=list(vacc)))
            return recs[-1]["id"]

        def wait(ev, F):
            """-> the record a wait orders after; a ring slot's wait is checked to still mark the block it means"""
            ring = EV[ev.ring]
            if ring in ("ev_main", "ev_urgent"):
                return F
            ops.append(("wait", ring, ev.slot, recs[tier_upto[ev.blk]]["q"] if ring == "ev_bs" else ev.blk))
            return marks.get((ring, ev.slot))

        for q in range(self.Q):
            # the fused kernel of block q (upper level: on the side stream, in order with the MAC)
            if p["tail_pf"] == 1:
                F = rec("M", "fused", q, [], [(allc, q, 0, p["mac_lo"])], (), [(allc, "Y", q, "read")] if q >= 1 else [])
            else:
                c = lib.fused_read(q)
                nps = np.array([lib.fused_parts(q, s) for s in range(C)]) if p["fold"] else p["mac_lo"]
                vacc = [(allc, b, q, "read") for b, i in (("V", c.v), ("Y", c.y)) if i >= 0]
                F = rec("F", "fused", q, [wait(c.wait, None)] if c.wait.ring else [], [(allc, q, 0, nps)], (), vacc)

            # what follows block q: the per-block MAC of period q + tail_pf or the merged grid, the tier launches
            steps = lib.tail_steps(q, C)
            made = []
            for x in steps.l[:steps.n]:
                sums, reads, vacc = [], [], []
                if x.kind != TIER:
                    sums.append((allc, x.j, p["mac_lo"], p["mac_hi"]))
                    reads.append((x.j - p["mac_hi"] + 1, x.j - p["mac_lo"]))
                    vacc += [(allc, b, x.j, m) for b, i, m in (("Y", x.y, "init"), ("V", x.v, "read")) if i >= 0]
                if x.kind != MAC:
                    self.tier_parts(q, x.d, sums, reads, vacc)
                kind = ("mac", "merged", "far" if x.d.tier else "near")[x.kind]
                r = rec(("M", "B")[x.role], kind, q, [wait(w, F) for w in x.wait if w.ring], sums, reads, vacc)
                if x.kind != MAC:
                    made.append(r)
                for e in x.rec:
                    if e.ring:
                        marks[(EV[e.ring], e.slot)] = r
                        ops.append(("rec", EV[e.ring], e.slot, e.blk))
            tier_upto.append(made[-1] if made else (tier_upto[-1] if tier_upto else None))
        return recs, ops


def _clocks(recs):
    """Vector clocks: clk[id][stream] = the last record of that stream ordered before record id starts."""
    clk, last = [], {}
    for r in recs:
        c = dict(clk[last[r["stream"]]]) if r["stream"] in last else {}
        if r["stream"] in last:
            c[r["stream"]] = last[r["stream"]]
        for w in r["waits"]:
            for k, v in clk[w].items():
                c[k] = max(c.get(k, -1), v)
            c[recs[w]["stream"]] = max(c.get(recs[w]["stream"], -1), w)
        clk.append(c)
        last[r["stream"]] = r["id"]
    return lambda a, b: a is not None and b is not None and clk[b].get(recs[a]["stream"], -1) >= a   # a before b


def check(sched, recs, ops):
    """-> {check number: [failures]} of the five checks."""
    P, Q, C = sched.P, sched.Q, sched.C
    before = _clocks(recs)
    bad = defaultdict(list)
    cnt = np.zeros((C, Q, P), dtype=np.int16)
    parts = np.arange(P)
    for r in recs:
        for ch, j, lo, hi in r["sums"]:
            if j < Q:
                cnt[ch, j, :] += (parts >= lo) & (parts < np.broadcast_to(hi, ch.shape)[:, None])
    due = parts[None, :] <= np.arange(Q)[:, None]
    for s, j, p in zip(*np.nonzero((cnt != 1) & due[None])):
        bad[1].append((int(s), int(j), int(p), int(cnt[s, j, p])))
    fused = {r["q"]: r["id"] for r in recs if r["kind"] == "fused"}
    acc = defaultdict(lambda: ([], [], []))
    for r in recs:
        if r["kind"] != "fused":
            for b0, b1 in r["reads"]:
                if b1 > r["q"]:
                    bad[2].append((r["id"], r["kind"], r["q"], b1))
                if 0 <= b0 + sched.R < Q and not before(r["id"], fused[b0 + sched.R]):
                    bad[3].append((r["id"], r["kind"], r["q"], b0))
        for ch, buf, j, mode in r["vacc"]:
            if j < Q:
                for s in ch.tolist():
                    acc[(buf, s, j)][("init", "acc", "read").index(mode)].append(r["id"])
    by_slot = defaultdict(list)
    for (buf, s, j) in acc:
        by_slot[(buf, s, j % sched.slots[buf])].append(j)
    for (buf, s, j), (inits, accs, reads) in acc.items():
        what = (buf, s, j)
        if len(inits) > 1 or (accs and not inits) or ((inits or accs) and not reads):
            bad[4].append(what + ("writers", len(inits), len(accs), len(reads)))
        if any(not before(i, a) for i in inits for a in accs) or any(not before(w, x) for w in inits + accs for x in reads):
            bad[4].append(what + ("read before write",))
        for j2 in by_slot[(buf, s, j % sched.slots[buf])]:
            if j2 != j:
                for w in acc[(buf, s, j2)][0] + acc[(buf, s, j2)][1]:
                    if not ((inits and before(w, inits[0])) or all(before(x, w) for x in reads + accs)):
                        bad[4].append(what + ("overwritten by period", j2))
    state = {}
    for op, ring, idx, label in ops:
        if op == "rec":
            state[(ring, idx)] = label
        elif state.get((ring, idx)) != label:
            bad[5].append((ring, idx, label, state.get((ring, idx))))
    return bad


@pytest.mark.parametrize("name", list(PLANS))
def test_fir_tier_schedule(lib, name):
    sched = Schedule(lib, *PLANS[name])
    if not sched.has_tail:
        pytest.skip("no tail, or the pipeline kernel's")
    recs, ops = sched.enumerate()
    bad = check(sched, recs, ops)
    assert not bad, (name, sched.p, {k: v[:4] for k, v in bad.items()})


@pytest.fixture(scope="module")
def headline(lib):
    sched = Schedule(lib, *PLANS["bench/headline"])
    recs, ops = sched.enumerate()
    assert sched.p["fold"] and sched.p["stagger"] and not check(sched, recs, ops)
    return sched, recs, ops


def _broken(headline, change):
    sched, recs, ops = headline
    recs, ops = copy.deepcopy(recs), list(ops)
    change(sched, recs, ops)
    return check(sched, recs, ops)


def _mid_fused(sched, recs):
    return next(r for r in recs if r["kind"] == "fused" and r["q"] == sched.Q // 2)


def test_breaks_exactly_once(headline):
    """One partition fewer in one fused-kernel record: that partition of that period is summed by nobody."""
    def drop(sched, recs, ops):
        r = _mid_fused(sched, recs)
        ch, j, lo, hi = r["sums"][0]
        hi = hi.copy()
        hi[5] -= 1
        r["sums"][0] = (ch, j, lo, hi)
    assert set(_broken(headline, drop)) == {1}


def test_breaks_slots(headline):
    """The fused kernel of one block waits for the tier launches one block earlier than tier_wait() says: its V_j is
    read before the launch after block j - la has written it."""
    def earlier(sched, recs, ops):
        r = _mid_fused(sched, recs)
        w = r["waits"][0]
        r["waits"] = [max(x["id"] for x in recs if x["stream"] == "B" and x["q"] < recs[w]["q"])]
    assert 4 in _broken(headline, earlier)


def test_breaks_fdl_reuse(headline):
    """The fused kernels from the middle on wait for the tier launches two blocks earlier than tier_wait() says: the
    launch after block j - la - 1 still reads the FDL row that block j overwrites (one block earlier is still covered
    through the fused kernel of block j - 1)."""
    def earlier2(sched, recs, ops):
        for r in recs:
            if r["kind"] == "fused" and r["q"] >= sched.Q // 2:
                r["waits"] = [max(x["id"] for x in recs if x["stream"] == "B" and x["q"] < recs[r["waits"][0]]["q"] - 1)]
    assert 3 in _broken(headline, earlier2)


def test_breaks_causality(headline):
    """One pass launch issued one block earlier, as if it followed the block before the newest one it reads."""
    def shift(sched, recs, ops):
        r = next(x for x in recs if x["stream"] == "B" and x["q"] == sched.Q // 2)
        r["q"] -= 1
    assert 2 in _broken(headline, shift)


def test_breaks_event_rings(headline):
    """One wait on the ev_bs ring uses the slot before the one recorded for the block it means."""
    def slot(sched, recs, ops):
        i = next(k for k, op in enumerate(ops) if op[0] == "wait" and op[1] == "ev_bs" and op[3] >= sched.Q // 2)
        op, ring, idx, label = ops[i]
        ops[i] = (op, ring, (idx - 1) % RINGS["ev_bs"], label)
    assert set(_broken(headline, slot)) == {5}
