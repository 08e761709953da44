// fir_plan.h -- K2: the FIR plan policy (which levels, tiers and kernel forms a FirOp uses) and the schedule each plan
// runs (which launch sums which partitions of which periods, and what it waits for): values chosen from the call's shape
// and the DSP_B200_FIR_* knobs, tested without a device; fir.cu allocates and launches what they say.
#pragma once
#include <cstdio>
#include <cstdlib>
#include <optional>
#include <string>
#include <utility>

#ifdef __CUDACC__
#define FIR_HD __host__ __device__ __forceinline__
#else
#define FIR_HD inline
#endif

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
	// folded tail: no per-block MAC; the fused kernel of block j starts from V_j and sums fir_fused_parts() partitions
	bool fold = false;
	// look-ahead of the folded near tier: its launch after block q covers the periods q+la .. q+la+T-1, from partition
	// la + t on for period q+la+t (every block involved is complete).  3 by default; 2 on the full-wave plan (below),
	// where the fused kernel is the step's critical path and one partition fewer per block shortens it.
	int la = 3;
	// mid-window pass (staggered full-wave plans with one tier, la = 2; DSP_B200_FIR_PASS=0|m, default T/2): the grid
	// launched after block q' also runs a pass for the class whose tier launch came after block q = q' - pass_m.  For
	// its periods q+la+t with t >= pass_m it adds partitions la+t-pass_m .. la-1+t to V in place (blocks q'-pass_m+1 ..
	// q'), and the fused kernel sums 0 .. la-1+t-pass_m there: la .. la-1+max(pass_m, T-pass_m) partitions instead of
	// la .. la-1+T.
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
	// partitions [first, second) of a tail-level period the per-block MAC sums: from tail_pf up to the near tier's start
	std::pair<int, int> mac_parts() const { return { tail_pf, (t_batch > 0) ? t_batch + tail_pf : lv[n_levels - 1].P }; }
	// The consumer of V_j (the fused kernel of block j when folded, else the per-block MAC of period j) is ordered after
	// the tier launches up to block tier_wait(j) (< 0: none); they run in order on one stream, a launch after block q once
	// the fused kernel of block q is complete.  T = t_batch.
	//  - folded: j-la.  V ring of 2T slots, T >= la: the next write to V_j's slot is for period j+2T, after block
	//    j+T-la+1 > j.  FDL row j mod P (X_{j-P}) is read by the launches up to block j-la-1; the pass after q' reads rows
	//    q'-pass_m+1 .. q', overwritten by blocks that wait for q'-pass_m+1+P-la >= q'.
	//  - per-block MAC: j-3, the launches before its own block j-2 (the fused kernel of block j waits for the MAC).
	//  - merged grid (merge_tail): the grids up to block j-2, one stream.  Upper level: the launch after T floor((j-2)/T).
	long tier_wait(long j) const
	{
		if (t_batch == 0) return -1;
		if (n_levels > 1) return (j >= 2) ? t_batch * ((j - 2) / t_batch) : -1;
		return j - (fold ? la : merge_tail ? 2 : 3);
	}
	// Slots of the tail level's spectrum rings: V of the near (tier 0) or far tier (1), Y; and the slot of period j
	int v_slots(int tier) const { return 2 * (tier ? t_far : t_batch); }
	int y_slots() const { return tail_pf; }
	int v_slot(long j) const { return (int) (j % v_slots(0)); }
	int y_slot(long j) const { return (int) (j % y_slots()); }
};

#ifdef __CUDA_ARCH__
FIR_HD int fir_log2(int w) { return __ffs(w) - 1; }   // w: a power of two
#else
FIR_HD int fir_log2(int w) { return __builtin_ctz(w); }
#endif

// Channels of a batch-tier launch: K classes take turns over groups of w adjacent channels (w a power of two; 0, 1, 1:
// all channels).  Row y of class g is channel (g + K (y / w)) w + y % w; class g has fir_class_rows() rows.
FIR_HD int fir_class_channel(int g, int K, int w, int y) { return ((g + K * (y >> fir_log2(w))) << fir_log2(w)) + (y & (w - 1)); }
inline int fir_class_rows(int n_sel, int g, int K, int w)
{
	int n = 0;
	for (int G = g; G * w < n_sel; G += K) n += (n_sel - G * w < w) ? n_sel - G * w : w;
	return n;
}

// Folded: the fused kernel of block j sums partitions 0 .. n-1 of channel s.  V_j came from its class's near-tier launch
// after block j-la-t, t = (j - la - class) mod T (partitions from la + t on); for t >= pass_m the pass after block
// j-la-t+pass_m <= j-la added la+t-pass_m .. la-1+t.  Before the class's first launch (d < 0) V_j is zero: np_max.
FIR_HD int fir_fused_parts(long blk, int s, int T, int K, int w, int la, int pass_m, int np_max)
{
	const long d = blk - la - (s >> fir_log2(w)) % K;
	if (d < 0) return np_max;
	int t = (int) (d % T);
	if (t >= pass_m) t -= pass_m;
	return la + t;
}

// The batch kernel's window for a launch after block q: FDL rows m in [pf+1, x_hi) hold X_{q+pf+1-m}; row m meets filter
// row m+t for period j = q+pf+1+t when p_lo <= m+t < h_hi; periods t < n_t are written.  Tier role: [p_lo, p_hi).  Pass
// role: blocks q-pass_m+1 .. q, filter rows < p_lo+T-1, the periods the tier launch after q-pass_m covered from t = pass_m.
struct FirBatchWindow { int x_hi, h_hi, n_t; };
FIR_HD FirBatchWindow fir_batch_window(bool pass, int T, int p_lo, int p_hi, int pass_m)
{
	return pass ? FirBatchWindow{ p_lo + pass_m, p_lo + T - 1, T - pass_m } : FirBatchWindow{ p_hi, p_hi, T };
}

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

// One batch-tier launch after block q of the tail level (k_fir_mac_batch, or the batch rows of k_fir_tail): V_j of the
// `rows` channels of class g for the periods j = q+pf+1+t (fir_batch_window), started from the far tier's V_j when
// from_far; pass_rows > 0: the same grid runs the mid-window pass of class pass_g (FirSchedule::pass_m).
struct FirTierLaunch {
	int tier;   // 0: near (V), 1: far (V2)
	int T, g, K, w, pf, p_lo, p_hi, rows;
	bool from_far;
	int pass_g, pass_rows, pass_m;
};
struct FirTierLaunches { int n = 0; FirTierLaunch l[2]; };

// The tier launches after block q of the tail level, far tier first (the near tier starts from its sums).  Each
// channel's periods are covered once: staggered, class (s / class_w) mod T every block, else all channels every T-th
// block (the far tier: far_classes classes in turns); a near window lies inside one far window (t_far is a multiple of
// t_batch).  Folded, period q+la+t gets every p >= la+t, the fused kernel the rest.  Upper level: all channels every
// T-th block, pf = 1.  A launch with no rows (fewer channels than classes) is listed but not made.
inline FirTierLaunches fir_tier_launches(const FirSchedule &s, long q, int n_sel)
{
	FirTierLaunches r;
	const int P = s.lv[s.n_levels - 1].P;
	if (s.t_batch == 0 || s.use_pipe) return r;
	for (int i = (s.t_far > 0) ? 1 : 0; i >= 0; --i) {
		const int T = i ? s.t_far : s.t_batch;
		const int K = s.stagger ? T : (i ? s.far_classes : 1), w = s.class_w, period = T / K;
		if (q % period != 0) continue;
		const int g = (int) ((q / period) % K), rows = fir_class_rows(n_sel, g, K, w);
		const bool pass = i == 0 && s.pass_m > 0 && q >= s.pass_m;
		const int gp = pass ? (int) ((q - s.pass_m) % K) : 0, prows = pass ? fir_class_rows(n_sel, gp, K, w) : 0;
		const int pf = i ? 2 + s.far_e : (s.tail_pf == 1) ? 1 : s.la - 1;
		const bool from_far = i == 0 && s.t_far > 0;
		r.l[r.n++] = { i, T, g, K, w, pf, (i == 0 && s.fold) ? s.la : T + pf, from_far ? s.t_far + 2 + s.far_e : P, rows, from_far,
		               gp, prows, prows > 0 ? s.pass_m : 0 };
	}
	return r;
}

// ---- The tail's cross-stream protocol; fir.cu maps its stream roles to streams and its slots to events and spectra.
enum FirEvRing { FIR_EV_NONE, FIR_EV_MAIN, FIR_EV_URGENT, FIR_EV_TAIL, FIR_EV_BATCH, FIR_EV_BS };
constexpr int FIR_N_EV_TAIL = 2, FIR_N_EV_BATCH = 2, FIR_N_EV_BS = 8, FIR_N_BS_AT = 4;
// ev_main / ev_urgent: the caller stream after block q / the side stream after the upper level's partition-0 kernels.
// blk: a label for tests/test_fir_tiers_cpu.py (fir.cu does not read it), the block (ev_tail: period) the event marks.
struct FirEv { int ring = FIR_EV_NONE, slot = 0; long blk = 0; };
// ev_bs records so far (record n >= 1 in slot (n - 1) mod FIR_N_EV_BS); folded, at[q mod FIR_N_BS_AT]: n after block q
struct FirTailRing { long n = 0; long at[FIR_N_BS_AT] = {}; };
inline int fir_bs_slot(long n) { return (int) ((n - 1) % FIR_N_EV_BS); }

enum FirTailKind { FIR_TAIL_MAC, FIR_TAIL_MERGED, FIR_TAIL_TIER };
enum FirTailRole { FIR_SIDE, FIR_SIDE2 };
struct FirTailStep {
	int kind = FIR_TAIL_MAC, role = FIR_SIDE;
	FirEv wait[2], rec[2];   // waited for before it (ev_main, ev_urgent first), recorded after it
	long j = 0;              // MAC, merged grid: Y_j into Y slot y, from V slot v (-1: zero)
	int y = -1, v = -1;
	FirTierLaunch d = {};    // tier launch; the merged grid's batch rows
};
struct FirTailSteps { int n = 0; FirTailStep l[3]; };

// The launches after block q of the tail level in issue order: unless folded, the per-block MAC of period q + tail_pf or
// the merged grid (side stream), then the tier launches that have rows (second side stream).
inline FirTailSteps fir_tail_steps(const FirSchedule &s, long q, int n_sel, FirTailRing &r)
{
	FirTailSteps o;
	if (s.tail_pf == 0 || s.use_pipe) return o;
	const bool l0 = s.tail_pf == 2;
	const long j = q + s.tail_pf, qw = s.tier_wait(j);
	const FirEv start = { l0 ? FIR_EV_MAIN : FIR_EV_URGENT, 0, q };
	auto batch = [&](long b) { return FirEv{ FIR_EV_BATCH, (int) ((b / s.t_batch) % FIR_N_EV_BATCH), b }; };
	auto bs_record = [&] { return FirEv{ FIR_EV_BS, (int) (r.n++ % FIR_N_EV_BS), q }; };
	const FirTierLaunches tl = fir_tier_launches(s, q, n_sel);
	if (!s.fold) {
		FirTailStep &m = o.l[o.n++];
		m.kind = s.merge_tail ? FIR_TAIL_MERGED : FIR_TAIL_MAC;
		m.j = j; m.y = s.y_slot(j); m.v = (s.t_batch > 0) ? s.v_slot(j) : -1;
		m.wait[0] = l0 ? start : (qw >= 0) ? batch(qw) : FirEv{};
		if (l0 && !s.merge_tail && r.n > 0) m.wait[1] = { FIR_EV_BS, fir_bs_slot(r.n), qw };
		if (l0) m.rec[0] = { FIR_EV_TAIL, (int) (j % FIR_N_EV_TAIL), j };
		if (s.merge_tail) { m.d = tl.l[0]; m.rec[1] = bs_record(); return o; }
	}
	const int first = o.n;   // the tier launches that have rows: the first waits for the block, the last records
	for (int i = 0; i < tl.n; ++i) {
		if (tl.l[i].rows + tl.l[i].pass_rows == 0) continue;
		FirTailStep &b = o.l[o.n++];
		b.kind = FIR_TAIL_TIER; b.role = FIR_SIDE2; b.d = tl.l[i];
	}
	if (o.n > first) { o.l[first].wait[0] = start; o.l[o.n - 1].rec[0] = l0 ? bs_record() : batch(q); }
	if (s.fold) r.at[q % FIR_N_BS_AT] = r.n;
	return o;
}

// What the fused kernel of block j (single level) waits for and starts from (-1: zero, as V_j before block tier_wait(j))
struct FirTailRead { FirEv wait; int y = -1, v = -1; };
inline FirTailRead fir_fused_read(const FirSchedule &s, long j, const FirTailRing &r)
{
	FirTailRead c;
	const long qw = s.tier_wait(j);
	if (s.fold && qw >= 0) {
		const long n = r.at[qw % FIR_N_BS_AT];
		c.v = s.v_slot(j);
		if (n > 0) c.wait = { FIR_EV_BS, fir_bs_slot(n), qw };
	}
	if (!s.fold && s.tail_pf == 2 && !s.use_pipe && j >= 2) { c.y = s.y_slot(j); c.wait = { FIR_EV_TAIL, (int) (j % FIR_N_EV_TAIL), j }; }
	return c;
}
// The general path's block j (single level) overwrites an FDL row the tier launches read: after every one so far
inline FirEv fir_general_wait(long j, const FirTailRing &r) { return (r.n > 0) ? FirEv{ FIR_EV_BS, fir_bs_slot(r.n), j - 1 } : FirEv{}; }

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
