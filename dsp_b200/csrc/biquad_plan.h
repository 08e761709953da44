// biquad_plan.h -- K1's host code, tested without a device: the per-stage scan table and the launch of each call.
#pragma once
#include <cmath>
#include <vector>

namespace dspb200 {

constexpr int BQ_L = 16;           // frames per lane
constexpr int BQ_MAX_STAGES = 16;  // stages fused into one operator
constexpr int BQ_NPOW = 6;         // M^(L 2^r), r = 0..5
// per channel and stage: 5 coefficients (+1 pad), BQ_NPOW 2x2 matrices M^(L 2^r), the basis T and T^-1 (2x2 each), and
// G[i] = T^-1 A^(L-1-i) B (2 x L), contiguous; every piece starts on a 16-byte boundary so that the kernel reads the
// table with 128-bit shared loads
constexpr double BQ_EPS_MIN = 1.0 / 32;
constexpr int BQ_OFF_P = 6, BQ_OFF_T = BQ_OFF_P + 4 * BQ_NPOW, BQ_OFF_G = BQ_OFF_T + 8;
constexpr int BQ_TBL = BQ_OFF_G + 2 * BQ_L;
static_assert(BQ_TBL % 2 == 0 && BQ_OFF_G % 2 == 0, "table pieces must stay 16-byte aligned");

// CH adjacent channels share a CTA; a warp's lanes are (32 / CH consecutive chunks) x (CH channels), channel
// fastest, so that one load instruction touches 32 / CH rows and uses CH x 8 contiguous bytes of each.
// SPLIT: two CTAs per channel pair, each on one half (2048 frames) of a 4096-frame tile, 8 warps each -- two of
// them fit an SM, so that one CTA's barriers, table loads and block I/O hide behind the other's arithmetic.  The
// second half needs, per stage, the state the first half ends in: the first half publishes it (state, fence, flag)
// as soon as its stage is done and the second half picks it up right before that stage's carry step, i.e. it runs
// one stage behind (decoupled look-back along time; CTAs of the first half have the lower block indices, so they
// are always scheduled before the CTAs that wait for them).
template <int CH, bool SPLIT = false>
struct BqCfg {
	static_assert(CH == 1 || CH == 2 || CH == 4, "1, 2 or 4 channels per CTA");
	static_assert(!SPLIT || CH == 2, "the split form is built for channel pairs");
	static constexpr int CPW = 32 / CH;                         // chunks per warp
	static constexpr int LOGW = (CH == 1) ? 5 : (CH == 2) ? 4 : 3;
	static constexpr int WARPS = SPLIT ? 8 : (CH == 1) ? 8 : 16;
	static constexpr int THREADS = 32 * WARPS;
	static constexpr long TILE = (long) BQ_L * CPW * WARPS;     // frames per tile
};

struct BqMat { long double a, b, c, d; };   // [[a, b], [c, d]]
struct BqVec { long double x, y; };
inline BqMat bq_mul(const BqMat &p, const BqMat &q) { return { p.a * q.a + p.b * q.c, p.a * q.b + p.b * q.d, p.c * q.a + p.d * q.c, p.c * q.b + p.d * q.d }; }
inline BqVec bq_apply(const BqMat &m, const BqVec &v) { return { m.a * v.x + m.b * v.y, m.c * v.x + m.d * v.y }; }
inline void bq_put(double *t, const BqMat &m) { t[0] = (double) m.a; t[1] = (double) m.b; t[2] = (double) m.c; t[3] = (double) m.d; }

// One stage's table t[BQ_TBL] from its coefficients cf[5]
inline void bq_stage_table(const double *cf, double *t)
{
	for (int k = 0; k < 6; ++k) t[k] = (k < 5) ? cf[k] : 0.0;   // the coefficients and the pad
	// A = [[-c3, 1], [-c4, 0]], B = (c1 - c3 c0, c2 - c4 c0): z' = A z + B s   (biquad.h:79-81 with r = c0 s + m0)
	const BqMat Az = { -(long double) cf[3], 1.0L, -(long double) cf[4], 0.0L };
	const BqVec Bz = { (long double) cf[1] - (long double) cf[3] * cf[0], (long double) cf[2] - (long double) cf[4] * cf[0] };
	// the scan's basis (biquad.cu header): z = T w, w' = M w + T^-1 B s
	const long double al = -(long double) cf[3] / 2, d2 = al * al - (long double) cf[4];
	long double eps = sqrtl(fabsl(d2));
	if (eps < BQ_EPS_MIN) eps = BQ_EPS_MIN;
	const BqMat T = { 1.0L, 0.0L, -al, eps }, Ti = { 1.0L, 0.0L, al / eps, 1.0L / eps }, M = bq_mul(Ti, bq_mul(Az, T));
	bq_put(t + BQ_OFF_T, T);
	bq_put(t + BQ_OFF_T + 4, Ti);
	// G[i] = M^(L-1-i) T^-1 B, i = L-1 .. 0
	BqVec g = bq_apply(Ti, Bz);
	for (int i = BQ_L - 1; i >= 0; --i, g = bq_apply(M, g)) {
		t[BQ_OFF_G + 2 * i] = (double) g.x;
		t[BQ_OFF_G + 2 * i + 1] = (double) g.y;
	}
	// M^L, then M^(L 2^r) by repeated squaring
	BqMat p = { 1.0L, 0.0L, 0.0L, 1.0L };
	for (int i = 0; i < BQ_L; ++i) p = bq_mul(M, p);
	for (int r = 0; r < BQ_NPOW; ++r, p = bq_mul(p, p)) bq_put(t + BQ_OFF_P + 4 * r, p);
}

// coefs [stage][channel][5] as handed in -> the kernel's [C][S][BQ_TBL] (a CTA reads its channels' tables)
inline std::vector<double> bq_table(int C, int S, const double *coefs)
{
	std::vector<double> tbl((size_t) C * S * BQ_TBL);
	for (int c = 0; c < C; ++c)
		for (int st = 0; st < S; ++st) bq_stage_table(&coefs[((size_t) st * C + c) * 5], &tbl[((size_t) c * S + st) * BQ_TBL]);
	return tbl;
}

// One call: `launches` launches of k_bq_cascade<ch, split> on `span` frames each (the last one may be shorter), on
// grid x (1 + split) CTAs of `threads`, with `smem` bytes of dynamic shared memory (the CTA's channel tables).
struct BqLaunch { int ch = 0, split = 0, threads = 0, grid = 0; size_t smem = 0; long span = 0, launches = 0; };

// force_ch: DSP_B200_BQ_CH (0 when unset); force_split: DSP_B200_BQ_SPLIT (-1 when unset: auto; 0 never, else always)
inline BqLaunch bq_launch(int C, int S, long frames, int force_ch, int force_split)
{
	BqLaunch L;
	// Channel pairs unless forced: the scan's association order depends on the chunks per warp, and a channel's
	// result must not depend on how the chain was sharded (tests: sharded == unsharded, bit for bit).
	L.ch = (force_ch == 0 || force_ch == 2) ? 2 : (force_ch == 4) ? 4 : 1;
	// Split form: slower than one 16-warp CTA on full tiles (the second half trails by a stage, and a pair's two CTAs
	// contend for one SM's FP64 pipe), but calls of at most 2048 frames have no second half: 8 warps beat 16 half-idle.
	L.split = L.ch == 2 && ((force_split >= 0) ? force_split != 0 : frames <= BqCfg<2, true>::TILE);
	L.threads = L.split ? BqCfg<2, true>::THREADS : (L.ch == 4) ? BqCfg<4>::THREADS : (L.ch == 2) ? BqCfg<2>::THREADS : BqCfg<1>::THREADS;
	L.grid = (C + L.ch - 1) / L.ch;
	L.smem = (size_t) L.ch * S * BQ_TBL * sizeof(double);
	L.span = L.split ? 2 * BqCfg<2, true>::TILE : frames;   // the split form: one launch per 4096-frame tile
	L.launches = L.split ? (frames + L.span - 1) / L.span : 1;
	return L;
}

}  // namespace dspb200
