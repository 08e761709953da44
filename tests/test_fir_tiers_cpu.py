"""CPU tier: the FIR tail schedule of dsp_b200/csrc/fir_plan.h, compiled with g++ alone.

For every plan with a tail (the pipeline kernel's aside) the whole-block schedule is enumerated from the header's
functions alone -- fir_tier_launches(), fir_batch_window(), fir_class_channel(), fir_fused_parts(),
FirSchedule::mac_parts() and FirSchedule::tier_wait() -- as the launches fir.cu makes: the fused kernel of every block
(one stream, in order), the per-block MAC or the merged grid (a side stream), the tier launches (a second side stream),
over enough blocks to pass start-up and wrap the V and FDL rings several times.  Then:

1. exactly once: every partition p <= j of every period j of every channel is summed by exactly one launch;
2. causality: a launch after block q reads only blocks <= q;
3. FDL reuse: a launch that reads block b is ordered before the fused kernel of block b + R, which overwrites its row;
4. V, V2 and Y slots: every write of a period is ordered before its readers, no write of another period of the slot
   lands in between, and every write is read (a reader that finds no write reads the zeros of an unwritten slot);
5. event rings: the event each wait uses still marks the block it means when the wait is enqueued.

"Ordered" follows from in-order streams, "a launch after block q starts after the fused kernel of block q" and the
wait rule tier_wait().  Each check is shown to fail on a broken copy of the headline's records.
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
extern "C" void plan(long taps, long hint, int n_sel, int sm_count, int *o)
{
	g = fir_schedule({ taps, hint, n_sel, sm_count, true, true }, FirKnobs::from_env());
	const FirLevelPlan &L = g.lv[g.n_levels - 1];
	const int v[] = { g.n_levels, L.P, L.R, g.tail_pf, g.t_batch, g.t_far, g.fold, g.stagger, g.merge_tail, g.use_pipe,
	                  g.mac_parts().first, g.mac_parts().second };
	for (int i = 0; i < 12; ++i) o[i] = v[i];
}
extern "C" int tier_launches(long q, int n_sel, int *o)   // 13 ints per launch
{
	const FirTierLaunches r = fir_tier_launches(g, q, n_sel);
	for (int i = 0; i < r.n; ++i) {
		const FirTierLaunch &d = r.l[i];
		const int v[] = { d.tier, d.T, d.g, d.K, d.w, d.pf, d.p_lo, d.p_hi, d.rows, d.from_far, d.pass_g, d.pass_rows, d.pass_m };
		for (int k = 0; k < 13; ++k) o[13 * i + k] = v[k];
	}
	return r.n;
}
extern "C" long tier_wait(long j) { return g.tier_wait(j); }
// as fir.cu's fused kernel gets it: K = T classes when staggered, else 1; at most l0_parts()
extern "C" int fused_parts(long blk, int s)
{
	return fir_fused_parts(blk, s, g.t_batch, g.stagger ? g.t_batch : 1, g.class_w, g.la, g.pass_m, g.l0_parts());
}
extern "C" void batch_window(int pass, int T, int p_lo, int p_hi, int pass_m, int *o)
{
	const FirBatchWindow w = fir_batch_window(pass != 0, T, p_lo, p_hi, pass_m);
	o[0] = w.x_hi; o[1] = w.h_hi; o[2] = w.n_t;
}
extern "C" int class_channel(int g_, int K, int w, int y) { return fir_class_channel(g_, K, w, y); }
"""
PLAN_KEYS = ("n_levels", "P", "R", "tail_pf", "t_batch", "t_far", "fold", "stagger", "merge", "pipe", "mac_lo", "mac_hi")
LAUNCH_KEYS = ("tier", "T", "g", "K", "w", "pf", "p_lo", "p_hi", "rows", "from_far", "pass_g", "pass_rows", "pass_m")
RINGS = dict(ev_bs=8, ev_bs_at=4, ev_batch=2, ev_tail=2)   # fir.cu's event rings


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = header_lib(tmp_path_factory.mktemp("fir_tiers"), "firtiers", DRIVER)
    lib.tier_wait.argtypes, lib.tier_wait.restype = [ctypes.c_long], ctypes.c_long
    lib.tier_launches.argtypes = [ctypes.c_long, ctypes.c_int, ctypes.c_void_p]
    lib.fused_parts.argtypes = [ctypes.c_long, ctypes.c_int]
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
        o = (ctypes.c_int * 12)()
        with env(**{k: None for k in os.environ if k.startswith("DSP_B200_FIR_")}):
            with env(**envs):
                lib.plan(ctypes.c_long(taps), ctypes.c_long(hint), C, SMS, o)
        self.lib, self.C = lib, C
        self.p = dict(zip(PLAN_KEYS, o))
        p = self.p
        self.has_tail = p["tail_pf"] > 0 and not p["pipe"]
        self.P, self.R = p["P"], p["R"]
        self.Q = 3 * self.P + 4 * max(p["t_batch"], p["t_far"], 1) + 4
        self.slots = dict(V=2 * p["t_batch"], V2=2 * p["t_far"], Y=p["tail_pf"])

    def launches(self, q):
        buf = (ctypes.c_int * 26)()
        n = self.lib.tier_launches(q, self.C, buf)
        return [dict(zip(LAUNCH_KEYS, buf[13 * i:13 * i + 13])) for i in range(n)]

    def window(self, pass_, d):
        o = (ctypes.c_int * 3)()
        self.lib.batch_window(int(pass_), d["T"], d["p_lo"], d["p_hi"], d["pass_m"], o)
        return tuple(o)

    def chans(self, g, K, w, rows):
        return np.array([self.lib.class_channel(g, K, w, y) for y in range(rows)], dtype=np.int64)

    def enumerate(self):
        """-> (records, ops).  A record is one launch: id, stream, kind, q (the block it follows; a fused kernel's own
        block), waits (ids it is ordered after), sums [(channels, period, first partition, end)], reads [(first block,
        last block)] of the FDL, vacc [(channels, buffer, period, "init" | "acc" | "read")].  ops: the host's event
        operations in issue order, ("rec" | "wait", ring, index, block or period it marks / must mark)."""
        p, lib, C = self.p, self.lib, self.C
        allc = np.arange(C)
        recs, ops = [], []
        mac_of = {}                   # period -> the record that writes its Y
        tier_upto = []                # tier_upto[q]: the last tier record issued after a block <= q
        bs_n, bs_last, bs_at = 0, None, [None] * RINGS["ev_bs_at"]
        multi = p["tail_pf"] == 1

        def rec(stream, kind, q, waits, sums=(), reads=(), vacc=()):
            recs.append(dict(id=len(recs), stream=stream, kind=kind, q=q, waits=[w for w in waits if w is not None],
                             sums=list(sums), reads=list(reads), vacc=list(vacc)))
            return recs[-1]["id"]

        def last_tier(qw):
            return tier_upto[qw] if 0 <= qw < len(tier_upto) else None

        def tier_parts(q):
            """-> [(tier, sums, reads, vacc)] of the tier launches after block q that have rows"""
            out = []
            for d in self.launches(q):
                sums, reads, vacc = [], [], []
                for pass_, g, rows in ((False, d["g"], d["rows"]), (True, d["pass_g"], d["pass_rows"])):
                    if rows == 0:
                        continue
                    ch = self.chans(g, d["K"], d["w"], rows)
                    x_hi, h_hi, n_t = self.window(pass_, d)
                    pf = d["pf"]
                    reads.append((q + pf + 1 - (x_hi - 1), q))   # FDL rows m in [pf+1, x_hi): X_{q+pf+1-m}
                    for t in range(n_t):
                        j = q + pf + 1 + t
                        sums.append((ch, j, max(pf + 1 + t, d["p_lo"]), min(x_hi + t, h_hi)))
                        if pass_:
                            vacc.append((ch, "V", j, "acc"))
                        else:
                            vacc.append((ch, "V2" if d["tier"] else "V", j, "init"))
                            if d["from_far"]:
                                vacc.append((ch, "V2", j, "read"))
                if sums:
                    out.append((d["tier"], sums, reads, vacc))
            return out

        for q in range(self.Q):
            # the fused kernel of block q (upper level: on the side stream, in order with the MAC)
            if multi:
                F = rec("M", "fused", q, [], [(allc, q, 0, p["mac_lo"])], (), [(allc, "Y", q, "read")] if q >= 1 else [])
            elif p["fold"]:
                qw = lib.tier_wait(q)
                nps = np.array([lib.fused_parts(q, s) for s in range(C)])
                if qw >= 0:
                    ops.append(("wait", "ev_bs_at", qw % RINGS["ev_bs_at"], qw))
                    if bs_at[qw % RINGS["ev_bs_at"]] is not None:
                        ops.append(("wait", "ev_bs", bs_at[qw % RINGS["ev_bs_at"]], recs[last_tier(qw)]["q"]))
                F = rec("F", "fused", q, [last_tier(qw)], [(allc, q, 0, nps)], (), [(allc, "V", q, "read")] if qw >= 0 else [])
            else:
                if q >= 2:
                    ops.append(("wait", "ev_tail", q % RINGS["ev_tail"], q))
                F = rec("F", "fused", q, [mac_of.get(q)], [(allc, q, 0, p["mac_lo"])], (), [(allc, "Y", q, "read")] if q >= 2 else [])

            # what follows block q: the per-block MAC of period q + tail_pf, the tier launches after block q
            j = q + p["tail_pf"]
            mac = ([(allc, j, p["mac_lo"], p["mac_hi"])], [(j - p["mac_hi"] + 1, j - p["mac_lo"])],
                   [(allc, "Y", j, "init")] + ([(allc, "V", j, "read")] if p["t_batch"] else []))
            made = []
            if p["merge"]:
                parts = tier_parts(q)
                sums, reads, vacc = (list(x) for x in mac)
                for _, s_, r_, v_ in parts:
                    sums += s_; reads += r_; vacc += v_
                mac_of[j] = rec("M", "merged", q, [F], sums, reads, vacc)
                made = [mac_of[j]]
            else:
                if not p["fold"]:
                    qw = lib.tier_wait(j)
                    if multi and qw >= 0:
                        ops.append(("wait", "ev_batch", (qw // p["t_batch"]) % RINGS["ev_batch"], qw))
                    if not multi and bs_last is not None:
                        ops.append(("wait", "ev_bs", bs_last, recs[last_tier(qw)]["q"]))
                    mac_of[j] = rec("M", "mac", q, [F, last_tier(qw)], *mac)
                for tier, s_, r_, v_ in tier_parts(q):
                    made.append(rec("B", "far" if tier else "near", q, [F], s_, r_, v_))
                if multi and made:
                    ops.append(("rec", "ev_batch", (q // p["t_batch"]) % RINGS["ev_batch"], q))
            if not multi and not p["fold"]:
                ops.append(("rec", "ev_tail", j % RINGS["ev_tail"], j))
            if made and not multi:
                bs_last = bs_n % RINGS["ev_bs"]
                bs_n += 1
                ops.append(("rec", "ev_bs", bs_last, q))
            if p["fold"]:
                bs_at[q % RINGS["ev_bs_at"]] = bs_last
                ops.append(("rec", "ev_bs_at", q % RINGS["ev_bs_at"], q))
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
