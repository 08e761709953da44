// biquad.cu -- K1: fused, time-parallel biquad cascade (one kernel, one read + one write of the block).
//
// Reference behaviour reproduced (/root/reference): biquad() biquad.h:76-92 (transposed direct form II),
// applied in place per channel by biquad_effect_run[_all] biquad.c:296-315 -- one pass over the block PER
// STAGE there; here a cascade of S stages is ONE operator.
//
// Per stage (biquad.h:79-81):   r = c0 s + m0;  m0' = m1 + c1 s - c3 r;  m1' = c2 s - c4 r
// i.e. the state z = (m0, m1) follows z' = A z + B s with A = [[-c3, 1], [-c4, 0]] (zero-input step).
// The per-sample recurrence is parallelised along TIME as an associative scan over these affine maps:
//   * a CTA owns two adjacent channels and a tile of 4096 frames; a lane owns one chunk of L = 16 frames of one
//     channel (a warp = 16 consecutive chunks x 2 channels, channel fastest), the chunk's samples live in
//     registers through all S stages;
//   * the scan runs in a better-conditioned basis w = T^-1 z (below); z is only formed for the re-run (4);
//   * per stage: (1) every lane needs the end state e its chunk would reach from a ZERO state; that is the
//     dot product e = sum_i A^(L-1-i) B s_i of the chunk with a per-stage table (2 L independent FMAs instead
//     of a serial recurrence; table built on the host in long double); (2) warp-level inclusive scan of the
//     states by shuffles -- all chunks share the matrix A^L, so round r is  s += A^(L 2^r) shfl_up(s, 2 * 2^r)
//     with the powers taken on the host in long double; (3) warp totals are chained through shared memory
//     with A^(16 L), every lane turns the carry-in of its warp into its own start state with the binary
//     expansion of its chunk index; (4) the lane re-runs the reference's own recurrence from that TRUE start
//     state -- so every output sample is produced by exactly the reference's arithmetic, started from a
//     state that differs from the sequential one by rounding in the scan (|eig A| < 1);
//   * longer calls loop over tiles, carrying the per-stage state through shared memory.
// Basis: with both poles near z = 1 (low corners at high rates: 10 Hz at 192 kHz) the companion matrix A is far from
// normal -- A^k has entries of order k that cancel to a state of order 1 -- and a scan on z loses about log2(k) bits,
// 50 to 150 times the sequential recurrence's own error.  With alpha = -c3 / 2 (the poles' mean) and
// eps = sqrt|alpha^2 - c4| (half their distance), T = [[1, 0], [-alpha, eps]] turns A into M = T^-1 A T =
// [[alpha, eps], [+-eps, alpha]]: symmetric for real poles, a scaled rotation for complex ones, normal either way, so
// the powers M^k stay bounded by 1 and the scan keeps the precision of its inputs.  eps is clamped below at 1/32 for
// (near-)double poles, where T would be singular; M is then only mildly non-normal.  Measured on the 10 Hz / 192 kHz
// sections the GPU lands within a few times the FP64 recurrence's error (tests/test_gpu_accuracy.py), on sections near
// Nyquist (poles near z = -1) at about that error (tests/test_gpu_dropin_effects.py; see step (1) below).
// A stage that does not act on a channel carries the identity section {1,0,0,0,0}.
// Global accesses: one load instruction of a warp touches 16 rows (frames) and uses 16 contiguous bytes of
// each -- half of every 32-byte sector, the neighbouring CTA uses the other half at about the same time, so
// HBM sees every sector once (L2 absorbs the rest).  (One channel per CTA = 32 sectors per request, slower than
// pairs; four channels per CTA halves the grid and loses more than it gains at 256 channels.)  Algorithmic bytes: 16 per sample.
#include "common.cuh"
#include "ops.h"
#include "biquad_plan.h"

namespace dspb200 {

struct M2 { double a, b, c, d; };  // [[a, b], [c, d]]

__device__ __forceinline__ double2 m2_apply(const M2 &m, double2 v)
{
	return make_double2(fma(m.a, v.x, m.b * v.y), fma(m.c, v.x, m.d * v.y));
}

struct BqSplitArgs {
	double *xstate;   // [C][S][2]: state at the end of the first half, per stage
	int *flag;        // [C][S]: == epoch once xstate[c][st] is valid
	int epoch;
};

// tbl: [C][S][BQ_TBL] (see BQ_TBL), zstate: [C][S][2]
template <int CH, bool SPLIT = false>
__global__ void __launch_bounds__(BqCfg<CH, SPLIT>::THREADS, SPLIT ? 2 : 1) k_bq_cascade(const double *in, double *out, const double *__restrict__ tbl,
                                                                  double *zstate, int C, int S, long frames, BqSplitArgs sp)
{
	using Cfg = BqCfg<CH, SPLIT>;
	const int half = SPLIT ? (int) blockIdx.y : 0;
	if (SPLIT && half == 1 && frames <= Cfg::TILE) return;   // nothing in the second half (the whole CTA leaves before any barrier)
	const bool second_exists = SPLIT && frames > Cfg::TILE;
	constexpr int LOGW = Cfg::LOGW;
	__shared__ double2 tot[Cfg::WARPS][CH];
	__shared__ double2 carry[BQ_MAX_STAGES][CH];
	extern __shared__ __align__(16) double stbl[];   // [CH][S][BQ_TBL]: these channels' tables
	const int c0 = blockIdx.x * CH;
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
	const int ch = lane & (CH - 1), jl = lane / CH;     // channel within the CTA, chunk within the warp
	const int c = c0 + ch;
	const bool have = c < C;
	const int nch = (C - c0 < CH) ? C - c0 : CH;
	for (int i = threadIdx.x; i < nch * S * BQ_TBL; i += blockDim.x) stbl[i] = tbl[(long) c0 * S * BQ_TBL + i];
	if (threadIdx.x < S * CH) {
		const int st = threadIdx.x / CH, k = threadIdx.x % CH;
		// (the second half's entries are filled stage by stage from the first half's published states)
		carry[st][k] = (k < nch && half == 0) ? make_double2(zstate[((long) (c0 + k) * S + st) * 2], zstate[((long) (c0 + k) * S + st) * 2 + 1])
		                                      : make_double2(0.0, 0.0);
	}
	__syncthreads();
	const double *mytbl = stbl + (have ? ch : 0) * S * BQ_TBL;

	for (long base = SPLIT ? half * Cfg::TILE : 0; base < frames; base += SPLIT ? frames : Cfg::TILE) {
		const long f0 = base + ((long) w * Cfg::CPW + jl) * BQ_L;
		const long rem = frames - f0;
		const int nv = (rem <= 0 || !have) ? 0 : (rem < BQ_L ? (int) rem : BQ_L);
		// the last valid chunk of this tile hands its end state to the next tile / the next call
		const bool last_chunk = nv > 0 && (rem <= BQ_L || f0 + BQ_L >= base + Cfg::TILE);
		double y[BQ_L];
#pragma unroll
		for (int i = 0; i < BQ_L; ++i) y[i] = (i < nv) ? in[(f0 + i) * C + c] : 0.0;

		for (int st = 0; st < S; ++st) {
			const double2 *t = reinterpret_cast<const double2 *>(mytbl + st * BQ_TBL);
			const double2 t0 = t[0], t1 = t[1], t2 = t[2];
			const double c0_ = t0.x, c1 = t0.y, c2 = t1.x, c3 = t1.y, c4 = t2.x;
			M2 P[LOGW + 1];
#pragma unroll
			for (int r = 0; r <= LOGW; ++r) {
				const double2 lo = t[BQ_OFF_P / 2 + 2 * r], hi = t[BQ_OFF_P / 2 + 2 * r + 1];
				P[r] = M2{ lo.x, lo.y, hi.x, hi.y };
			}
			// (1) zero-state end state of a FULL chunk as a dot product (a partial last chunk is nobody's predecessor:
			//     its value is never used; missing samples are zeros).  Two accumulators for ILP, each over consecutive
			//     frames (the first and the second half of the chunk): near Nyquist G alternates in sign, and splitting
			//     the terms into even and odd frames would build two large sums that cancel at the end -- 4 to 8 times
			//     the FP64 recurrence's error on a smooth input (tests/test_gpu_dropin_effects.py); in order, the
			//     partial sums stay as small as the terms.
			const double2 *G = t + BQ_OFF_G / 2;
			double ex0 = 0.0, ex1 = 0.0, ey0 = 0.0, ey1 = 0.0;
#pragma unroll
			for (int i = 0; i < BQ_L / 2; ++i) {
				const double2 g0 = G[i], g1 = G[i + BQ_L / 2];
				ex0 = fma(g0.x, y[i], ex0);
				ey0 = fma(g0.y, y[i], ey0);
				ex1 = fma(g1.x, y[i + BQ_L / 2], ex1);
				ey1 = fma(g1.y, y[i + BQ_L / 2], ey1);
			}
			// (2) inclusive scan over the chunks of this warp (uniform matrix A^L per chunk); lanes CH apart
			double2 sc = make_double2(ex0 + ex1, ey0 + ey1);
#pragma unroll
			for (int r = 0; r < LOGW; ++r) {
				const double vx = __shfl_up_sync(0xffffffffu, sc.x, CH << r), vy = __shfl_up_sync(0xffffffffu, sc.y, CH << r);
				if (jl >= (1 << r)) {
					const double2 u = m2_apply(P[r], make_double2(vx, vy));
					sc.x += u.x;
					sc.y += u.y;
				}
			}
			// exclusive: state at the start of this lane's chunk if the warp started from zero
			double2 z = make_double2(__shfl_up_sync(0xffffffffu, sc.x, CH), __shfl_up_sync(0xffffffffu, sc.y, CH));
			if (jl == 0) z = make_double2(0.0, 0.0);
			if (jl == Cfg::CPW - 1) tot[w][ch] = sc;
			if (SPLIT && half == 1 && w == 0 && jl == 0 && have) {
				// the state the first half left this stage in: wait for its flag, then read it past L1
				const long o = (long) c * S + st;
				volatile int *fl = sp.flag + o;
				while (*fl != sp.epoch) { }
				__threadfence();
				carry[st][ch] = make_double2(__ldcg(&sp.xstate[o * 2]), __ldcg(&sp.xstate[o * 2 + 1]));
			}
			__syncthreads();
			// (3) carry into this warp, then into this lane (the carried state is a true z: into the scan's basis)
			const double2 tb0 = t[BQ_OFF_T / 2], tb1 = t[BQ_OFF_T / 2 + 1], ti0 = t[BQ_OFF_T / 2 + 2], ti1 = t[BQ_OFF_T / 2 + 3];
			double2 cin = m2_apply(M2{ ti0.x, ti0.y, ti1.x, ti1.y }, carry[st][ch]);
			for (int k = 0; k < w; ++k) {
				const double2 u = m2_apply(P[LOGW], cin);
				cin = make_double2(u.x + tot[k][ch].x, u.y + tot[k][ch].y);
			}
#pragma unroll
			for (int r = 0; r < LOGW; ++r)
				if ((jl >> r) & 1) cin = m2_apply(P[r], cin);
			const double2 zs = m2_apply(M2{ tb0.x, tb0.y, tb1.x, tb1.y }, make_double2(z.x + cin.x, z.y + cin.y));
			double m0 = zs.x, m1 = zs.y;
			// (4) the real run from the true start state
#pragma unroll
			for (int i = 0; i < BQ_L; ++i) {
				if (i < nv) {
					const double s = y[i];
					const double r = c0_ * s + m0;
					m0 = m1 + c1 * s - c3 * r;
					m1 = c2 * s - c4 * r;
					y[i] = r;
				}
			}
			__syncthreads();   // everyone has read tot[] and carry[st]
			if (last_chunk) {
				carry[st][ch] = make_double2(m0, m1);
				if (SPLIT && half == 0 && second_exists) {
					const long o = (long) c * S + st;
					sp.xstate[o * 2] = m0;
					sp.xstate[o * 2 + 1] = m1;
					__threadfence();
					*reinterpret_cast<volatile int *>(sp.flag + o) = sp.epoch;
				}
			}
		}
#pragma unroll
		for (int i = 0; i < BQ_L; ++i)
			if (i < nv) out[(f0 + i) * C + c] = y[i];
		__syncthreads();   // carry[] complete before the next tile reads it
	}
	if (threadIdx.x < S * CH && (!SPLIT || half == 1 || !second_exists)) {   // the CTA that holds the end of the block
		const int st = threadIdx.x / CH, k = threadIdx.x % CH;
		if (k < nch) {
			zstate[((long) (c0 + k) * S + st) * 2] = carry[st][k].x;
			zstate[((long) (c0 + k) * S + st) * 2 + 1] = carry[st][k].y;
		}
	}
}

struct BiquadOp : Op {
	int S = 0;
	std::vector<double> h_coefs;   // [S][C][5] as handed in (kept so neighbouring cascades can be fused)
	double *d_tbl = nullptr, *d_zstate = nullptr;
	double *d_xstate = nullptr;   // split form: per-stage state between the two halves of a tile
	int *d_flag = nullptr;
	int epoch = 0;
	bool ran = false;   // d_zstate may hold state: run() since construction or the last reset()
	BqLaunch last;   // the last call's launches (describe(): ch = 0 before the first call)

	const char *name() const override { return "biquad"; }
	std::string describe() const override
	{
		char buf[96];
		snprintf(buf, sizeof(buf), "{\"op\":\"biquad\",\"stages\":%d,\"ch\":%d,\"split\":%d}", S, last.ch, last.split);
		return buf;
	}
	~BiquadOp() override { dev_free(d_tbl); dev_free(d_zstate); dev_free(d_xstate); dev_free(d_flag); }

	void reset(cudaStream_t st) override
	{
		cudaMemsetAsync(d_zstate, 0, (size_t) channels * S * 2 * sizeof(double), st);
		ran = false;
	}

	long run(long frames, const double *in, double *out, cudaStream_t st) override
	{
		if (frames <= 0) return 0;
		ran = true;
		ProfScope prof("biquad", st);
		static const int force_ch = getenv("DSP_B200_BQ_CH") ? atoi(getenv("DSP_B200_BQ_CH")) : 0;
		static const int force_split = getenv("DSP_B200_BQ_SPLIT") ? atoi(getenv("DSP_B200_BQ_SPLIT")) : -1;
		last = bq_launch(channels, S, frames, force_ch, force_split);
		const auto k_bq = last.split ? k_bq_cascade<2, true> : (last.ch == 4) ? k_bq_cascade<4> : (last.ch == 2) ? k_bq_cascade<2> : k_bq_cascade<1>;
		for (long i = 0, base = 0; i < last.launches; ++i, base += last.span) {
			const BqSplitArgs sp = last.split ? BqSplitArgs{ d_xstate, d_flag, ++epoch } : BqSplitArgs{};
			LAUNCH(k_bq, dim3(last.grid, 1 + last.split), last.threads, last.smem, st, in + base * channels, out + base * channels, d_tbl, d_zstate,
			       channels, S, (frames - base < last.span) ? frames - base : last.span, sp);
		}
		return frames;
	}
};

Op *make_biquad_op(int slab_channels, int fs, int n_stages, const double *coefs)
{
	if (n_stages < 1 || n_stages > BQ_MAX_STAGES) {
		set_error("biquad: %d stages per operator unsupported (1..%d)", n_stages, BQ_MAX_STAGES);
		return nullptr;
	}
	std::unique_ptr<BiquadOp> op(new BiquadOp());
	const int C = slab_channels, S = n_stages;
	op->channels = C; op->fs_in = op->fs_out = fs; op->S = S;
	op->h_coefs.assign(coefs, coefs + (size_t) S * C * 5);

	const std::vector<double> tbl = bq_table(C, S, coefs);
	op->d_tbl = dev_alloc<double>(tbl.size(), false);
	op->d_zstate = dev_alloc<double>((size_t) C * S * 2, true);
	op->d_xstate = dev_alloc<double>((size_t) C * S * 2, true);
	op->d_flag = dev_alloc<int>((size_t) C * S, true);
	if (!op->d_tbl || !op->d_zstate || !op->d_xstate || !op->d_flag) return nullptr;
	CUDA_TRY(cudaMemcpy(op->d_tbl, tbl.data(), tbl.size() * sizeof(double), cudaMemcpyHostToDevice), return nullptr);
	return op.release();
}

// Two adjacent cascades over the same slab become one operator (one pass over the block).  The fused
// operator starts from zero state, so cascades that have run since their last reset() are not fused.
Op *fuse_biquad_ops(Op *a, Op *b)
{
	BiquadOp *x = dynamic_cast<BiquadOp *>(a), *y = dynamic_cast<BiquadOp *>(b);
	if (!x || !y || x->ran || y->ran || x->channels != y->channels || x->fs_in != y->fs_in || x->S + y->S > BQ_MAX_STAGES) return nullptr;
	std::vector<double> all(x->h_coefs);
	all.insert(all.end(), y->h_coefs.begin(), y->h_coefs.end());
	return make_biquad_op(x->channels, x->fs_in, x->S + y->S, all.data());
}

}  // namespace dspb200
