// fir_plan.h -- K2: the FIR plan policy (which levels, tiers and kernel forms a FirOp uses), host-only: a value chosen
// from the call's shape and the DSP_B200_FIR_* knobs, tested without a device; fir.cu allocates and launches what it says.
#pragma once
#include <cstdio>
#include <cstdlib>
#include <optional>
#include <string>

namespace dspb200 {

constexpr int FIR_MAX_LEVELS = 8;
constexpr int FIR_MAX_B = 8192;
constexpr int FIR_NB_MAX = 8;       // whole blocks per bulk launch (k_fir_mac_bulk)
constexpr int FIR_T_BATCH = 4;      // default depth of the near tier; DSP_B200_FIR_T=4|6|8|12 selects an instantiation
constexpr int FIR_T_FULL_WAVE = 8;  // ... on full-wave plans of at least 2 * 8 + 3 partitions
constexpr int FIR_T_FAR = 8;        // default depth of the far tier (DSP_B200_FIR_T2=0|8|12|16) ...
constexpr int FIR_FAR_MIN_P = 48;   // ... on levels of at least this many partitions
constexpr int PIPE_TB = 4;          // batch depth of the pipeline kernel (fir_pipe.cuh): outputs per pass, = channel residues

inline bool batch_depth_ok(int T) { return T == 4 || T == 6 || T == 8 || T == 12 || T == 16; }
inline bool pipe_size_ok(int N) { return N == 2048 || N == 4096; }
// channels per CTA of the FFT kernels, FftCfg<N>::CPB (fir.cu checks that the two agree)
constexpr int fir_fft_cpb(int N) { return (N / 16 >= 256) ? 1 : 256 / (N / 16); }

// The DSP_B200_FIR_* knobs a plan reads; from_env() is the only place they are parsed.  Unset: empty / default.
struct FirKnobs {
	long level_cap = 4096, single_min = 2048;
	bool no_bulk = false, pipe = false, hot = true, no_batch = false, merge = false, pipe_stats = false;
	std::optional<int> t, t2, far_classes, pass, mac_prio;
	std::optional<bool> stagger, fold;

	static FirKnobs from_env()
	{
		auto env = [](const char *k) { return getenv((std::string("DSP_B200_FIR_") + k).c_str()); };
		auto on = [&](const char *k) { const char *e = env(k); return e && e[0] == '1'; };
		FirKnobs k;
		if (const char *e = env("LEVEL_CAP")) k.level_cap = atol(e);
		if (const char *e = env("SINGLE_MIN")) k.single_min = atol(e);
		k.no_bulk = on("NO_BULK"); k.pipe = on("PIPE"); k.no_batch = on("NO_BATCH"); k.merge = on("MERGE");
		k.hot = !(env("HOT") && env("HOT")[0] == '0'); k.pipe_stats = env("PIPE_STATS") != nullptr;
		if (const char *e = env("T")) k.t = (atoi(e) == 12) ? 12 : (atoi(e) == 8) ? 8 : (atoi(e) == 6) ? 6 : 4;
		if (const char *e = env("T2")) k.t2 = atoi(e);
		if (const char *e = env("FAR_CLASSES")) k.far_classes = atoi(e);
		if (const char *e = env("PASS")) k.pass = atoi(e);
		if (const char *e = env("MAC_PRIO")) k.mac_prio = atoi(e);
		if (const char *e = env("STAGGER")) k.stagger = e[0] != '0';
		if (const char *e = env("FOLD")) k.fold = e[0] == '1';
		return k;
	}
};

// What a plan depends on besides the knobs (whether the channels share one filter does not change it)
struct FirShape {
	long filter_frames = 0, hint = 0;   // hint: frames of the call (or the caller's block hint) the plan is made for
	int n_sel = 0, sm_count = 0;
	bool multilevel = true, direct_io = true;   // !DSP_B200_FIR_LEVELS=1, !DSP_B200_FIR_NO_DIRECT=1 (read when the operator is made)
};

struct FirLevelPlan {
	int B = 0, P = 0, R = 0;      // R: rows of the FDL ring per channel (P, or more when calls bring several blocks at once)
	long tap0 = 0, tap1 = 0;      // taps [tap0, tap1) of the filter
	// last level only: partitions p >= 1 ("tail") are summed by the MAC kernels on a side stream, one block
	// period ahead, into a spectrum that the level's partition-0 kernel adds before its inverse transform
	bool tail = false;
};

struct FirSchedule {
	int B0 = 0, n_levels = 0;
	FirLevelPlan lv[FIR_MAX_LEVELS];
	// bulk form (single-level plans): up to nb_max whole blocks of one call are transformed, multiplied and
	// overlapped by one launch each
	int nb_max = 1;
	int tail_pf = 0;              // 0: no tail; 1: tail on an upper level; 2: tail on level 0 (single-level plan, fused kernel sums p = 0, 1)
	// time-batched tail (see k_fir_mac_batch): V spectra for 2 T block periods, produced T at a time on a second side stream
	int t_batch = 0;
	// single-level plans: a second, deeper tier over the oldest partitions (its sums are the near tier's starting value);
	// `stagger`: every block launches the tiers for one residue class of channels instead of all every T-th block
	int t_far = 0;
	// The far tier works one near-tier period ahead: launched after block q it covers the periods q+3+far_e .. (partitions
	// >= t_far + 2 + far_e), so that the step time does not hang on how fast one whole-launch far tier runs.
	int far_e = 0;
	// Far tier in whole launches: far_classes residue classes of channels take turns, one launch every t_far /
	// far_classes blocks (DSP_B200_FIR_FAR_CLASSES=2: half the channels every fourth block at t_far = 8)
	int far_classes = 1;
	bool stagger = false;
	bool merge_tail = false;      // the per-block MAC and the staggered batch launch as one grid (k_fir_tail)
	// single-level plans of 2048/4096-frame blocks: whole aligned blocks go through the persistent pipeline
	// (fir_pipe.cuh), which sums partitions 0 .. pipe_pf-1 (+ the batched V) itself -- no per-block k_fir_mac
	bool use_pipe = false;
	int pipe_pf = 0;
	// folded tail: the fused kernel of block j starts from V_j, which the tier launches up to block j-la complete
	bool fold = false;
	// look-ahead of the folded near tier: its launch after block q covers the periods q+la .. q+la+T-1, from partition
	// la + t on for period q+la+t (every block involved is complete).  3 by default; 2 on the full-wave plan (below),
	// where the fused kernel is the step's critical path and one partition fewer per block shortens it.
	// Invariants (T = t_batch):
	//  - the V ring of 2 T slots is safe for T >= la: the next write to V_j's slot is for period j + 2T, by a launch after
	//    block j + T - la + 1 > j or later, and launches only start once the fused kernel of their block is complete;
	//  - FDL row j mod P (X_{j-P} until block j overwrites it) is read by the tier launches after blocks up to j-la-1;
	//    the fused kernel of block j waits for the launches up to j-la, which covers them;
	//  - the general path (wait_batch_for) still waits for every launch made so far.
	int la = 3;
	// mid-window pass (staggered full-wave plans with one tier, la = 2; DSP_B200_FIR_PASS=0|m, default T/2): the grid
	// launched after block q' also runs a pass for the class whose tier launch came after block q = q' - pass_m.  For
	// its periods q+la+t with t >= pass_m it adds partitions la+t-pass_m .. la-1+t to V in place (blocks q'-pass_m+1 ..
	// q'), and the fused kernel sums 0 .. la-1+t-pass_m there: la .. la-1+max(pass_m, T-pass_m) partitions instead of
	// la .. la-1+T.  Invariants, in addition to those of `la`:
	//  - the pass after q' reads X_{q'} and waits for the fused kernel of block q', like the tier launch after q';
	//  - the fused kernel of block j = q+la+t, t >= pass_m, waits for the launches up to j-la = q+t >= q', the pass included;
	//  - V slots: the pass touches the periods q+la+pass_m .. q+la+T-1; the class's next tier launch (after q+T) writes
	//    q+T+la .. q+2T+la-1: disjoint in the ring of 2T slots; their next writer, the tier launch after q+2T, comes after
	//    the fused kernels that read them;
	//  - FDL: the pass reads only rows newer than the tier launch of the same grid does (q'-pass_m+1 .. q'); the first
	//    block to overwrite one, q'-pass_m+1+P, waits for the launches up to q'-pass_m+1+P-la >= q' (P >= 2T+3).
	int pass_m = 0;
	// staggered folded plans: the classes take turns over groups of class_w adjacent channels (1 otherwise), so that
	// the four channels of a cluster sum the same number of partitions and finish together
	int class_w = 1;
	// single-level tail plans: the fused kernel of every block goes to a stream of the highest priority, so that its CTAs
	// are placed before the queued CTAs of the look-ahead MACs (the lowest priority, shared with a caller's default stream)
	bool hot = false;
	long hist_len = 0; int Bmax = 0;   // frames of the history ring per channel; the largest partition

	// partitions level 0's fused kernel sums on whole aligned blocks: at most, and (folded: once every class has had a
	// near-tier launch) at least
	int l0_parts() const { return fold ? t_batch + la - 1 : (lv[0].P < 2) ? lv[0].P : 2; }
	int l0_parts_min() const { return fold ? la : l0_parts(); }
	// at most, once every class has had its mid-window pass (l0_parts() without one)
	int l0_parts_steady() const { return fold ? la - 1 + ((pass_m > t_batch - pass_m) ? pass_m : t_batch - pass_m) : l0_parts(); }
};

inline FirSchedule fir_schedule(const FirShape &sh, const FirKnobs &k)
{
	FirSchedule s;
	s.B0 = 64;
	while (s.B0 * 2 <= sh.hint && s.B0 < FIR_MAX_B) s.B0 *= 2;
	const long T = sh.filter_frames;
	// level plan (fir.cu's header).  Partitions grow up to `cap`: beyond it the larger transforms cost more than the
	// filter traffic they save once the tail is time-batched (DESIGN.md K2)
	long cap = k.level_cap;
	if (cap < s.B0) cap = s.B0;
	if (cap > FIR_MAX_B) cap = FIR_MAX_B;
	// Blocks of 2048 frames stay a single level: fewer bytes per sample than 2048 + 4096 (544 against 612 at 131072
	// taps), and no upper-level kernel that has to land between two blocks
	s.lv[0].B = s.B0; s.n_levels = 1;
	if (!sh.multilevel || T <= 2L * s.B0 || s.B0 >= cap || s.B0 >= k.single_min) s.lv[0].tap1 = T;
	else {
		s.lv[0].tap1 = 2L * s.B0;
		long B = 2L * s.B0;
		while (s.n_levels < FIR_MAX_LEVELS) {
			FirLevelPlan &L = s.lv[s.n_levels++];
			L.B = (int) B; L.tap0 = B;
			if (B >= cap || T <= 2 * B || s.n_levels == FIR_MAX_LEVELS) { L.tap1 = T; break; }
			L.tap1 = 2 * B;
			B *= 2;
		}
	}
	for (int l = 0; l < s.n_levels; ++l) {
		FirLevelPlan &L = s.lv[l];
		L.P = (int) ((L.tap1 - L.tap0 + L.B - 1) / L.B);
		L.R = L.P;
		if (s.n_levels == 1 && L.P > 2 && sh.hint >= 2L * L.B && !k.no_bulk) {
			s.nb_max = (int) ((sh.hint / L.B < FIR_NB_MAX) ? sh.hint / L.B : FIR_NB_MAX);
			L.R = L.P + s.nb_max - 1;
		}
	}
	s.Bmax = s.lv[s.n_levels - 1].B;
	// upper levels read their block from the ring on the side stream while the next block is already
	// being stashed: keep two of the largest blocks
	s.hist_len = (s.n_levels > 1) ? 2L * s.Bmax : (long) s.nb_max * s.Bmax;

	// the last level's partitions beyond those its fused kernel sums form the "tail"; a single level keeps
	// partitions 0 and 1 in the kernel (pf = 2), an upper level only partition 0 (pf = 1)
	FirLevelPlan &L = s.lv[s.n_levels - 1];
	const bool l0 = s.n_levels == 1;
	const int pf = l0 ? 2 : 1;
	L.tail = L.P > pf && (!l0 || (s.nb_max == 1 && sh.multilevel));
	if (!L.tail) return s;
	s.tail_pf = pf;
	// the pipeline kernel is opt-in: slower than the three-kernel step on the headline (DESIGN.md K2)
	s.use_pipe = l0 && sh.direct_io && pipe_size_ok(L.B) && k.pipe;
	s.hot = !s.use_pipe && l0 && sh.direct_io && k.hot;
	// The fold pays once the fused kernel's CTAs outnumber half the SMs (see `fold` below).  Those plans are
	// "full-wave": the fused kernel fills the GPU and carries most of the bytes, so the near tier goes deeper
	// (T = 8 reads every FDL and filter row once per 8 periods instead of 4: 440 -> 388 B/sample on the
	// headline) and, with one tier, looks two blocks ahead instead of three (la = 2: 360 B/sample).
	const int cpb = fir_fft_cpb(L.B);
	const bool fold_pays = 2 * ((sh.n_sel + cpb - 1) / cpb) > sh.sm_count;
	const bool full_wave = l0 && !s.use_pipe && sh.direct_io && fold_pays;
	int tb = (full_wave && L.P >= 2 * FIR_T_FULL_WAVE + pf + 1) ? FIR_T_FULL_WAVE : FIR_T_BATCH;
	if (k.t) tb = *k.t;
	if (s.use_pipe) tb = PIPE_TB;   // the pipeline kernel's batch depth is compiled in (one channel residue per block)
	if (L.P >= 2 * tb + pf + 1 && !k.no_batch) {
		s.t_batch = tb;
		if (!s.use_pipe && pf == 2) {
			// far tier: partitions >= t_far + 2, T = t_far periods per launch, where it pays: not at 32 partitions, at 64
			// behind a near tier of 4; on the full-wave plan one staggered tier of 8 is faster than tiers 4 + 8 and 8 + 16
			// (DESIGN.md K2)
			int t2 = (L.P >= FIR_FAR_MIN_P) ? FIR_T_FAR : 0;
			if (k.t2) t2 = *k.t2;
			if (!batch_depth_ok(t2) || t2 <= tb || t2 % tb != 0 || L.P < 2 * t2 + pf + tb) t2 = 0;
			if (t2 > 0) { s.t_far = t2; s.far_e = tb; }
			// one tier: staggered (every block period carries the same launches); two tiers, or a tail too short for
			// per-class launches to pay (config 5's 16 partitions): whole launches
			s.stagger = k.stagger ? *k.stagger : (s.t_far == 0 && L.P - tb - pf >= 16);
			if (s.t_far > 0 && !s.stagger) {
				// the turns must start on near-tier launches (one turn by default: two were no faster at 2048 frames)
				const int fcls = k.far_classes.value_or(1);
				s.far_classes = (fcls >= 1 && s.t_far % fcls == 0 && (s.t_far / fcls) % tb == 0) ? fcls : 1;
			}
			// (opt-in: the fused kernel of the block after next would wait for all of the grid: a slower step)
			s.merge_tail = s.stagger && s.t_far == 0 && tb == 4 && L.B >= 256 && k.merge;
		}
	}
	if (s.use_pipe) s.pipe_pf = (s.t_batch > 0) ? s.t_batch + 2 : L.P;
	// Folded tail: no per-block MAC, no Y spectrum through HBM (DESIGN.md K2).  Only when the fused kernel's CTAs
	// outnumber half the SMs: with fewer, the per-block MAC streams on the SMs the fused kernel leaves idle (64 channels
	// of 4096 frames: 8% slower folded, 256: 6% faster).  The look-ahead of 2 is for full-wave plans with one tier only.
	s.fold = l0 && !s.use_pipe && sh.direct_io && s.t_batch > 0 && !s.merge_tail && k.fold.value_or(fold_pays);
	s.la = (s.fold && full_wave && s.t_far == 0) ? 2 : 3;
	// the mid-window pass halves the fused kernel's triangle (see `pass_m`): 360 -> 334 B/sample on the headline
	if (s.fold && s.stagger && s.la == 2) {
		s.pass_m = k.pass.value_or(s.t_batch / 2);
		if (s.pass_m < 0 || s.pass_m >= s.t_batch) s.pass_m = 0;
	}
	// classes of up to 4 adjacent channels (a cluster's four when every class can have a whole group): a cluster that
	// finishes early hands its SMs to the queued batch CTAs at once instead of waiting for its slowest channel
	if (s.fold && s.stagger) {
		const int most = (sh.n_sel / s.t_batch < 4) ? sh.n_sel / s.t_batch : 4;
		while (s.class_w * 2 <= most) s.class_w *= 2;
	}
	return s;
}

// the schedule's part of FirOp::describe()
inline std::string fir_schedule_json(const FirSchedule &s)
{
	std::string j = "\"levels\":[";
	for (int l = 0; l < s.n_levels; ++l) j += (l ? ",{\"B\":" : "{\"B\":") + std::to_string(s.lv[l].B) + ",\"P\":" + std::to_string(s.lv[l].P) + "}";
	char buf[512];
	snprintf(buf, sizeof(buf), "],\"t_batch\":%d,\"t_far\":%d,\"far_e\":%d,\"far_classes\":%d,\"stagger\":%d,\"class_width\":%d,\"merge\":%d,\"tail_pf\":%d,"
	         "\"l0_parts\":%d,\"l0_parts_min\":%d,\"l0_parts_steady\":%d,\"lookahead\":%d,\"pass_m\":%d,\"bulk\":%d,\"pipe\":%d,\"pipe_pf\":%d",
	         s.t_batch, s.t_far, s.far_e, s.far_classes, s.stagger ? 1 : 0, s.class_w, s.merge_tail ? 1 : 0, s.tail_pf, s.l0_parts(),
	         s.l0_parts_min(), s.l0_parts_steady(), s.la, s.pass_m, s.nb_max, s.use_pipe ? 1 : 0, s.pipe_pf);
	return j + buf;
}

}  // namespace dspb200
