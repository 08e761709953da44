// fir.cu -- K2: FFT convolution engine behind `fir`, `fir_p` and `hilbert`.
//
// Reference behaviour reproduced (file:line in /root/reference):
//   fir_p_effect_run  fir_p.c:127-181   out = in * h, zero latency, any frames per call
//   fir_effect_run    fir.c:109-149     out = (in * h) delayed by len frames
//   fir_direct_effect_run fir.c:43-62   out = in * h, zero latency (short filters)
// The reference's partition plan (32-tap direct head + <=4 FFT groups on worker threads,
// fir_p.c:290-335) is a CPU latency device; its output is exactly the linear convolution, which is
// what is kept.
//
// GPU formulation.  Overlap-add with a frequency-domain delay line (FDL) per selected channel; the filter
// is cut into LEVELS whose partition size doubles from the call's block size B0 up to 4096 (a single level
// when B0 is already that large; DSP_B200_FIR_LEVEL_CAP moves the cap):
//   level 0: partition B0 (power of two <= 8192), advanced on every block of B0 frames
//   level l: partition B_l = 2^l B0, taps [B_l, 2 B_l), advanced whenever B_l frames have accumulated; its
//            result for block J is due when block J completes and is added during the next period ("pend")
//   the last level takes all remaining taps in P partitions.
// For one level with partition B:  X_j = RFFT_2B([x_j | 0]) -> FDL slot j mod R
//                                  S_j = sum_{p<P} X_{j-p} . H_p
//                                  s_j = IRFFT_2B(S_j); y_j = s_j[0:B) + carry; carry = s_j[B:2B)
// Who computes what:
//   k_fir_level0<B,P>   ONE kernel per level and block: forward transform, spectrum into the FDL, the first
//                       pf = P partitions of S_j from registers, + Y_j (below), inverse transform, overlap.
//                       On single-level plans it reads the caller's interleaved block and writes the caller's
//                       result itself (clusters of four adjacent channels share the rows through DSMEM); with a
//                       batch tier it starts from V_j and sums the partitions the tier left out ("folded": no
//                       k_fir_mac; fir_fused_parts() in fir_plan.h, which holds the whole schedule).
//   k_fir_mac           Y_j = V_j + sum_{pf<=p<pf+T} X_{j-p} . H_p on a side stream, a block period ahead (the
//                       blocks it needs were complete pf periods ago): the HBM-streaming kernel
//   k_fir_mac_batch<T>  V_j = sum_{p>=pf+T} X_{j-p} . H_p for T periods at once (filter rows slide through a
//                       register window: every FDL and filter row is read once per T outputs); folded, the near
//                       tier also takes every partition p < pf+T whose block is complete (the triangle p >= la+t);
//                       on the full-wave plan the same grid runs a mid-window pass (FirSchedule::pass_m)
//   k_fir_mac_bulk<8>   calls that bring several whole 8192-blocks: all partitions of up to 8 new blocks in
//                       one pass, with one forward and one inverse launch (k_fir_fwd / k_fir_inv, gridDim.y)
//   k_fir_stash/unstash interleaved <-> per-channel copies for multi-level plans and ragged calls
// Spectra are stored "packed": B complex per row, bin 0 = (DC.re, Nyquist.re); rows are 16 B bytes
// long, 128-byte aligned.  131072 taps, 4096-frame blocks: 1040 algorithmic bytes per sample for the plain
// uniform scheme, 508 with the fused kernel + per-block MAC + time-batched tail, 476 with the per-block MAC folded
// into the fused kernel, 440 with the near tier taking the triangle of partitions its rows already meet, 360 on the
// full-wave plan (256 channels fill the GPU with fused CTAs: a near tier of depth 8 that looks two blocks ahead), 334
// with the mid-window pass (the fused kernel sums 2 .. 5 partitions instead of 2 .. 9).
//
// Calls that are not whole aligned blocks take the general path, exact for ANY frames-per-call
// pattern: with R_j = sum_{1<=p<P0} X_{j-p} . H_p (completed level-0 blocks only)
//   out_j[m] = IRFFT(R_j)[m] + carry_{j-1}[m] + pend(m) + sum_{r<=m} x_j[r] h[m-r]
// i.e. a time-domain head over the samples of the still-incomplete block (k_fir_head) on top of the
// precomputed contribution of everything that is complete.  Levels >= 1 never need a head: they only
// ever look at completed blocks.  All paths share {history, FDLs, carries, block counters}.
#include "common.cuh"
#include "fft.cuh"
#include "fir_pipe.cuh"
#include "fir_plan.h"
#include "fir_tile.cuh"
#include "ops.h"
#include "../../include/dsp_b200.h"
#include <cooperative_groups.h>

namespace dspb200 {

std::atomic<int> g_fir_serialize{0};   // dspb200_debug_serialize(): no side streams (isolated kernel timings)

// dspb200_debug_stall(): a FirOp puts a delay kernel on each selected stream of its blocks blk % period == phase, right
// before that stream's first FIR launch of the block, so that the stream falls behind the others.  Packed in one word
// (roles | microseconds << 8 | period << 24 | phase << 44), read with one relaxed load per block; 0: off.
std::atomic<unsigned long long> g_fir_stall{0};
constexpr int FIR_STALL_MAX_US = 5000;

struct FirStall {
	int roles = 0, us = 0;
	long period = 1, phase = 0;
	static FirStall load()
	{
		const unsigned long long w = g_fir_stall.load(std::memory_order_relaxed);
		FirStall s;
		if (!w) return s;
		s.roles = (int) (w & 0xff); s.us = (int) ((w >> 8) & 0xffff); s.period = (long) ((w >> 24) & 0xfffff); s.phase = (long) (w >> 44);
		return s;
	}
	bool hits(int role, long blk) const { return (roles & role) && blk % period == phase; }
};

template <int... N> constexpr bool fft_cpb_matches() { return ((fir_fft_cpb(N) == FftCfg<N>::CPB) && ...); }
static_assert(fft_cpb_matches<64, 128, 256, 512, 1024, 2048, 4096, 8192>(), "fir_plan.h's fir_fft_cpb() is FftCfg<N>::CPB");

// ------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------

// interleaved block -> per-channel contiguous history ring; tile transpose through shared memory
__global__ void __launch_bounds__(256) k_fir_stash(const double *__restrict__ in, long stride, const int *__restrict__ ch_map,
                                                   double *__restrict__ hist, long hist_len, long pos, int frames, int n_sel)
{
	__shared__ double tile[32][33];
	const int f0 = blockIdx.x * 32, s0 = blockIdx.y * 32;
	const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
#pragma unroll
	for (int r = ty; r < 32; r += 8) {
		const int f = f0 + r, s = s0 + tx;
		tile[r][tx] = (f < frames && s < n_sel) ? in[(long) f * stride + ch_map[s]] : 0.0;
	}
	__syncthreads();
#pragma unroll
	for (int r = ty; r < 32; r += 8) {
		const int s = s0 + r, f = f0 + tx;
		if (s < n_sel && f < frames) hist[(long) s * hist_len + pos + f] = tile[tx][r];
	}
}

struct PendArgs {
	int n;
	const double *buf[FIR_MAX_LEVELS];   // [s][len]
	int len[FIR_MAX_LEVELS];
	int off[FIR_MAX_LEVELS];             // offset of this call's first frame inside the level's period
};

// per-channel contiguous result (+ pending contributions of the larger levels) -> interleaved block
__global__ void __launch_bounds__(256) k_fir_unstash(const double *__restrict__ y, long y_len, PendArgs pend, double *__restrict__ out,
                                                     long stride, const int *__restrict__ ch_map, int frames, int n_sel)
{
	__shared__ double tile[32][33];
	const int f0 = blockIdx.x * 32, s0 = blockIdx.y * 32;
	const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
	for (int r = ty; r < 32; r += 8) {
		const int s = s0 + r, f = f0 + tx;
		double v = 0.0;
		if (s < n_sel && f < frames) {
			v = y[(long) s * y_len + f];
			for (int l = 0; l < pend.n; ++l) v += pend.buf[l][(long) s * pend.len[l] + pend.off[l] + f];
		}
		tile[r][tx] = v;
	}
	__syncthreads();
#pragma unroll
	for (int r = ty; r < 32; r += 8) {
		const int f = f0 + r, s = s0 + tx;
		if (f < frames && s < n_sel) out[(long) f * stride + (ch_map ? ch_map[s] : s)] = tile[tx][r];
	}
}

struct FwdArgs {
	const double *in;       // per-channel contiguous source
	long ch_stride;         // elements between channels (0: one shared channel)
	long valid;             // frames available (<= B); the rest is zero
	double2 *spec;          // destination rows
	long spec_ch_stride;    // double2 elements between channels
	int slot;               // row within the channel
	const double2 *tw, *ptw;   // split twiddles W_2N^k, per-pass butterfly twiddles
	int n_ch;
	// bulk form (gridDim.y > 1): block i = blockIdx.y reads the ring at (ring_off + i N) % ring_len and
	// writes row (slot + i) % slot_rows; ring_len == 0: plain form
	long ring_len, ring_off;
	int slot_rows;
};

template <int N>
__global__ void __launch_bounds__(FftCfg<N>::THREADS) k_fir_fwd(FwdArgs a)
{
	extern __shared__ double2 smem[];
	constexpr int T = FftCfg<N>::T, CPB = FftCfg<N>::CPB;
	const int g = threadIdx.x / T, t = threadIdx.x % T;
	const int s = blockIdx.x * CPB + g;
	const bool active = s < a.n_ch;
	double2 *buf = smem + (size_t) g * FftCfg<N>::STRIDE;

	if (active) {
		const double *xs = a.in + (long) s * a.ch_stride;
		if (a.ring_len > 0) xs += (a.ring_off + (long) blockIdx.y * N) % a.ring_len;
		const bool aligned = ((reinterpret_cast<size_t>(xs) & 15) == 0);
		const double2 *x = reinterpret_cast<const double2 *>(xs);
		for (int n = t; n < N / 2; n += T) {
			double2 v;
			if (aligned && 2L * n + 1 < a.valid) v = x[n];
			else v = make_double2((2L * n < a.valid) ? xs[2 * n] : 0.0, (2L * n + 1 < a.valid) ? xs[2 * n + 1] : 0.0);
			buf[spad(n)] = v;
			buf[spad(n + N / 2)] = make_double2(0.0, 0.0);
		}
	}
	__syncthreads();
	fft_forward_smem<N>(buf, a.ptw, t);
	if (active) {
		const int slot = (a.ring_len > 0) ? (a.slot + (int) blockIdx.y) % a.slot_rows : a.slot;
		double2 *X = a.spec + (long) s * a.spec_ch_stride + (long) slot * N;
		// every thread owns the 8 bin pairs (k, N-k), k = t + i T; thread 0 also owns k = 0 and k = N/2
		double2 w[8];
#pragma unroll
		for (int i = 0; i < 8; ++i) w[i] = __ldg(&a.tw[t + i * T]);
#pragma unroll
		for (int i = 0; i < 8; ++i) {
			const int k = t + i * T;
			if (k == 0) {
				const double2 z0 = buf[0], zh = buf[spad(N / 2)];
				X[0] = make_double2(z0.x + z0.y, z0.x - z0.y);
				X[N / 2] = cconj(zh);   // E = Re z, O = Im z, w = -i
			}
			else {
				const double2 zk = buf[spad(k)], zn = buf[spad(N - k)];
				const double2 e = make_double2(0.5 * (zk.x + zn.x), 0.5 * (zk.y - zn.y));
				const double2 o = make_double2(0.5 * (zk.y + zn.y), -0.5 * (zk.x - zn.x));
				const double2 wo = cmul(w[i], o);
				X[k] = cadd(e, wo);
				X[N - k] = cconj(csub(e, wo));
			}
		}
	}
}

enum { INV_OUT = 1, INV_UPDATE_CARRY = 2, INV_RAW = 4 };
// INV_RAW (bulk form, block i = blockIdx.y): Y, out and carry are [i][s][N]-strided arrays; out gets the first
// half of the inverse transform and carry the second half, nothing is added (k_fir_unstash_bulk overlaps them)

struct InvArgs {
	const double2 *Y;       // [s][N] packed spectra
	double *out;            // INV_OUT: out[s * out_ch_stride + i] = first half + carry, i < B
	long out_ch_stride;     // even
	double *carry;          // [s][B]
	int flags;
	const double2 *tw, *ptw;
	int n_ch;
};

template <int N>
__global__ void __launch_bounds__(FftCfg<N>::THREADS) k_fir_inv(InvArgs a)
{
	extern __shared__ double2 smem[];
	constexpr int T = FftCfg<N>::T, CPB = FftCfg<N>::CPB;
	const int g = threadIdx.x / T, t = threadIdx.x % T;
	const int s = blockIdx.x * CPB + g;
	const bool active = s < a.n_ch;
	double2 *buf = smem + (size_t) g * FftCfg<N>::STRIDE;

	const long boff = (a.flags & INV_RAW) ? (long) blockIdx.y * a.n_ch : 0;   // bulk form: rows of block i
	if (active) {
		const double2 *Y = a.Y + (boff + s) * N;
		double2 yk[8], yn[8], w[8];
#pragma unroll
		for (int i = 0; i < 8; ++i) {
			const int k = t + i * T;
			yk[i] = Y[k];
			yn[i] = Y[(k == 0) ? N / 2 : N - k];
			w[i] = __ldg(&a.tw[k]);
		}
#pragma unroll
		for (int i = 0; i < 8; ++i) irfft_merge<N>(buf, t + i * T, N - (t + i * T), yk[i], yn[i], w[i]);
	}
	__syncthreads();
	fft_forward_smem<N>(buf, a.ptw, t);
	if (active) {
		const double scale = 1.0 / N;
		double2 *carry = reinterpret_cast<double2 *>(a.carry + (boff + s) * N);
		double2 *out = reinterpret_cast<double2 *>(a.out + (boff + s) * a.out_ch_stride);
		double2 c[8];
		if (a.flags & INV_RAW) {
#pragma unroll
			for (int i = 0; i < 8; ++i) {
				const int n = t + i * T;
				const double2 lo = buf[spad(n)], hi = buf[spad(n + N / 2)];
				out[n] = ola_scaled(lo, scale);
				carry[n] = ola_scaled(hi, scale);
			}
			return;
		}
		if (a.flags & INV_OUT) {
#pragma unroll
			for (int i = 0; i < 8; ++i) c[i] = carry[t + i * T];
		}
#pragma unroll
		for (int i = 0; i < 8; ++i) {
			const int n = t + i * T;
			const double2 lo = buf[spad(n)], hi = buf[spad(n + N / 2)];
			if (a.flags & INV_OUT) out[n] = ola_out(lo, scale, c[i]);
			if (a.flags & INV_UPDATE_CARRY) carry[n] = ola_scaled(hi, scale);
		}
	}
}

// Level 0 in one kernel when it has at most two partitions (P = 2 whenever larger levels exist):
// forward transform of the new block, its spectrum into the FDL, S = X_j H_0 + sum_{p>=1} X_{j-p} H_p
// formed by the thread that owns the bin pair (k, N-k) straight from registers, inverse transform in
// the same shared-memory buffer, overlap-add epilogue.  One launch instead of three and no spectrum
// round trip through HBM.
struct L0Args {
	const double *in;        // per-channel contiguous block (history ring)
	long in_ch_stride;
	double2 *fdl;            // [s][fdl_ch_stride], rows of N
	long fdl_ch_stride;      // rows per channel * N
	int fdl_rows;            // rows per channel (slot arithmetic)
	const double2 *H;        // [s or 0][rows][N]
	long h_ch_stride;
	int P, slot;             // P: partitions summed (1, 2: compiled in; more: the folded tail, k_fir_level0<N, 0>)
	// folded tail (cls_T > 0): block blk sums fir_fused_parts() partitions of channel s
	long blk;
	int cls_T, cls_K, cls_w, la, pass_m;
	double *out;             // [s][out_ch_stride]: first half + carry
	long out_ch_stride;
	double *carry;           // [s][N]
	const double2 *tw, *ptw;
	int n_ch;
	const double2 *init;     // [s][N] spectrum added to S before the inverse transform (NULL: none)
	// direct form (single-level plans): read the block from / write the result to the caller's interleaved
	// buffers instead of the per-channel staging copies (no stash / unstash kernels)
	const double *xin;       // NULL: use `in`
	long xin_stride;
	const int *xin_map;      // channel of selected channel s (NULL: s)
	double *yout;            // NULL: use `out`
	long yout_stride;
	const int *yout_map;
	int cluster_io;          // host: launch the CL variant (4 adjacent channels per cluster; needs xin and yout)
};

// FIR_L0_ASYNC: the cluster form of the fused kernel exchanges its samples between the CTAs of a cluster with bulk
// copies shared memory -> a neighbour's shared memory that complete bytes on the RECEIVER's mbarrier
// (cp.async.bulk.shared::cluster.shared::cta), instead of plain distributed-shared-memory stores fenced by
// cluster.sync().  The releasing cluster barrier compiles to MEMBAR.ALL.GPU (+ ERRBAR): every thread waits for all its
// global stores and prefetches in flight, four times per block; a third of the kernel's stall samples were that wait
// Here nobody fences: a CTA de-interleaves its rows into a staging area, one thread
// sends each channel's chunk (8.5 KB, already in the padded layout of the transform buffer) to its owner, and a CTA
// waits on its own mbarrier until the bytes addressed to it have landed.  (Per-element st.async -- 16 bytes and one
// transaction-count update on the receiver's mbarrier each -- is slower than the fenced form.)  0 selects the fenced
// form.
#ifndef FIR_L0_ASYNC
#define FIR_L0_ASYNC 1
#endif

template <int N>
struct L0ClCfg {
	static constexpr int CPB = FftCfg<N>::CPB;
	static constexpr int NCL = (CPB <= 2) ? 4 / CPB : 1;   // CTAs per cluster
	static constexpr int NPC = N / 2 / NCL;                // packed frame pairs a CTA moves for all four channels
	static constexpr int CHUNK = NPC + NPC / 16;           // the same, in the padded layout of the transform buffers (spad())
	// Staging (this CTA's rows of all four channels: on the way in what it read, on the way out what it is about to
	// write) = the SECOND halves of its transform buffers, which hold exactly 4 chunks: they are zeros on the way in
	// (filled after the exchange) and the new carry on the way out (stored before the exchange).  A separate 34 KB
	// staging area cost more than the fences it saved: the kernel runs 2 CTAs per SM and lives on what is left of
	// the L1 (padding its shared memory alone slows it down).  After the buffers: two mbarriers.
	static constexpr size_t SMEM = FIR_L0_ASYNC ? FftCfg<N>::SMEM + 16 : FftCfg<N>::SMEM;
};

// CL: launched as clusters of 4 / CPB CTAs = 4 ADJACENT channels (four CTAs of one 4096- or 8192-point transform, two
// CTAs of two 2048-point transforms) that do the direct-form I/O together: every CTA reads
// its share of the rows for all four channels (32 contiguous bytes per row: whole sectors, 128-bit loads) and
// drops each channel's samples into its owner's transform buffer through distributed shared memory; results
// travel back the same way.  (One channel per CTA reads 8 of every 32-byte sector it touches: slower than staged
// per-channel copies.)
#ifndef FIR_L0_MAXNREG
#define FIR_L0_MAXNREG 128
#endif
// P: partitions summed, or 0: a run-time count of at most a.P (single-level plans with a batch tier: the "folded" tail,
// fir_fused_parts(), so that no per-block MAC and no Y spectrum round trip are needed)
template <int N, int P, bool CL = false>
__global__ void __launch_bounds__(FftCfg<N>::THREADS) __maxnreg__((N == 4096) ? FIR_L0_MAXNREG : 128) k_fir_level0(L0Args a)
{
	extern __shared__ double2 smem[];
	constexpr int T = FftCfg<N>::T, CPB = FftCfg<N>::CPB;
	static_assert(!CL || CPB <= 2, "cluster I/O: four adjacent channels in 4 / CPB CTAs");
	constexpr int NCL = CL ? 4 / CPB : 1;          // CTAs per cluster
	constexpr int NPC = N / 2 / NCL;               // packed frame pairs a CTA moves for all four channels
	constexpr int THREADS = FftCfg<N>::THREADS;
	const int g = threadIdx.x / T, t = threadIdx.x % T;
	const int s = blockIdx.x * CPB + g;
	const bool active = s < a.n_ch;
	double2 *buf = smem + (size_t) g * FftCfg<N>::STRIDE;
	namespace cg = cooperative_groups;
	unsigned crank = 0;
#if FIR_L0_ASYNC
	constexpr int CHUNK = NPC + NPC / 16;
	constexpr unsigned CHUNK_BYTES = CHUNK * sizeof(double2);
	// staging chunk c (channel c of the cluster's four): the second half of a transform buffer holds NCL chunks
	auto stage = [&](int c) -> double2 * { return smem + (size_t) (c / NCL) * FftCfg<N>::STRIDE + spad(N / 2) + (size_t) (c % NCL) * CHUNK; };
	uint64_t *mbar = reinterpret_cast<uint64_t *>(reinterpret_cast<char *>(smem) + FftCfg<N>::SMEM);   // [0]: samples in, [1]: results in
	if constexpr (CL) {
		cg::cluster_group cluster = cg::this_cluster();
		crank = cluster.block_rank();
		if (threadIdx.x == 0) {
			mbar_init(&mbar[0], 1);
			mbar_init(&mbar[1], 1);
			asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
			mbar_arrive_expect_tx(&mbar[0], CPB * NCL * CHUNK_BYTES);   // the first half of this CTA's transform buffers
			mbar_arrive_expect_tx(&mbar[1], 4 * CHUNK_BYTES);           // this CTA's rows of all four channels
		}
		cluster.sync();   // mbarriers armed, every CTA running (nothing in flight yet: this fence is free)
	}
#else
	double2 *rbuf[4] = { buf, buf, buf, buf };
	if constexpr (CL) {
		cg::cluster_group cluster = cg::this_cluster();
		crank = cluster.block_rank();
#pragma unroll
		for (int c = 0; c < 4; ++c) rbuf[c] = cluster.map_shared_rank(smem + (size_t) (c % CPB) * FftCfg<N>::STRIDE, c / CPB);
		cluster.sync();   // a CTA's shared memory may only be touched once that CTA is known to be running
	}
#endif

	if (active) {
		double2 v[8];
		if constexpr (CL) {
			const int s0 = ((int) blockIdx.x - (int) crank) * CPB;
			const double *xr = a.xin + (a.xin_map ? a.xin_map[s0] : s0);
#pragma unroll
			for (int i = 0; i < NPC / THREADS; ++i) {
				const int n = (int) crank * NPC + (int) threadIdx.x + i * THREADS;
				const double *r0 = xr + 2L * n * a.xin_stride, *r1 = r0 + a.xin_stride;
				const double2 a0 = *reinterpret_cast<const double2 *>(r0), a1 = *reinterpret_cast<const double2 *>(r0 + 2);
				const double2 b0 = *reinterpret_cast<const double2 *>(r1), b1 = *reinterpret_cast<const double2 *>(r1 + 2);
#if FIR_L0_ASYNC
				const int nl = spad((int) threadIdx.x + i * THREADS);   // within this CTA's rows; its first row is a multiple of 16
				stage(0)[nl] = make_double2(a0.x, b0.x);
				stage(1)[nl] = make_double2(a0.y, b0.y);
				stage(2)[nl] = make_double2(a1.x, b1.x);
				stage(3)[nl] = make_double2(a1.y, b1.y);
#else
				rbuf[0][spad(n)] = make_double2(a0.x, b0.x);
				rbuf[1][spad(n)] = make_double2(a0.y, b0.y);
				rbuf[2][spad(n)] = make_double2(a1.x, b1.x);
				rbuf[3][spad(n)] = make_double2(a1.y, b1.y);
#endif
			}
		}
		else if (a.xin) {
			// frames 2n, 2n+1 of this channel: 8-byte loads one row apart (the 3 neighbouring channels' CTAs use the
			// rest of each sector at about the same time: L2 serves them)
			read_frame_pairs<T>(v, a.xin + (a.xin_map ? a.xin_map[s] : s), a.xin_stride, t);
		}
		else {
			const double2 *x = reinterpret_cast<const double2 *>(a.in + (long) s * a.in_ch_stride);
#pragma unroll
			for (int i = 0; i < 8; ++i) v[i] = x[t + i * T];
		}
		if constexpr (!(CL && FIR_L0_ASYNC)) fill_buf<N, T>(buf, CL ? nullptr : v, t);
	}
#if FIR_L0_ASYNC
	if constexpr (CL) {
		fence_proxy_async_smem();
		__syncthreads();
		if (threadIdx.x == 0) {
			// channel c of the four lives in CTA c / CPB, transform buffer c % CPB; this CTA's rows start at crank * NPC
			const uint32_t mb = smem_u32(&mbar[0]);
#pragma unroll
			for (int c = 0; c < 4; ++c) {
				const uint32_t dst = smem_u32(smem + (size_t) (c % CPB) * FftCfg<N>::STRIDE + spad((int) crank * NPC));
				bulk_s2c(mapa_u32(dst, c / CPB), smem_u32(stage(c)), CHUNK_BYTES, mapa_u32(mb, c / CPB));
			}
		}
		mbar_wait_cluster(&mbar[0], 0);   // the samples of this CTA's channels, from every CTA of the cluster
		// every CTA has everything <=> every copy out of a staging area is complete: the second halves become zeros
		cluster_barrier_relaxed();
		fill_buf<N, T>(buf, nullptr, t);
		__syncthreads();
	}
	else __syncthreads();
#else
	if constexpr (CL) cg::this_cluster().sync();
	else __syncthreads();
#endif
	if (active) {
		// what the middle and the last phase will read from HBM: start it moving towards L2 now, so that it
		// arrives while the first transform runs (the CTA's warps all sit in the same phase, nothing else hides it).
		// After the barrier: its release fence would wait for these requests too.
		const double2 *Hc = a.H + (long) s * a.h_ch_stride;
		if constexpr (P > 0) {
			const double2 *fc_ = a.fdl + (long) s * a.fdl_ch_stride;
			prefetch_rows(Hc, (long) P * N * sizeof(double2), t, T);
#pragma unroll
			for (int p = 1; p < P; ++p) prefetch_rows(fc_ + (long) ring_back(a.slot, p, a.fdl_rows) * N, (long) N * sizeof(double2), t, T);
			prefetch_rows(a.carry + (long) s * N, (long) N * sizeof(double), t, T);
			if (a.init) prefetch_rows(a.init + (long) s * N, (long) N * sizeof(double2), t, T);
		}
		else {
			// The folded tail reads 2 a.P rows and more per channel, and one wave of CTAs sums them in step: rows pulled
			// ahead evict the rows being summed (measured: a prefetch of partitions 0 and 1 here and of partition p+1
			// during partition p made the step 17% slower than this).  Only H_0, read right after the transform.
			prefetch_rows(Hc, (long) N * sizeof(double2), t, T);
		}
	}
	fft_forward_smem<N>(buf, a.ptw, t);
	if (active) {
		double2 *fdl = a.fdl + (long) s * a.fdl_ch_stride;
		const double2 *H = a.H + (long) s * a.h_ch_stride;
		double2 *X = fdl + (long) a.slot * N;
		const double2 *init = a.init ? a.init + (long) s * N : nullptr;
		const bool per_ch_h = a.h_ch_stride != 0;
		// (1) real split: X[k], X[N-k] to the FDL and, in place of Z, to shared memory.
		//     Thread t owns the pairs k = t + i T; thread 0 also owns k = 0 (packed DC/Nyquist) and k = N/2.
		//     (The twiddles are loaded again for the merge below: 32 registers that phase (2) has better use for.)
		double2 w[8];
#pragma unroll
		for (int i = 0; i < 8; ++i) w[i] = __ldg(&a.tw[t + i * T]);
#pragma unroll
		for (int i = 0; i < 8; ++i)
			rfft_split<N>(buf, t + i * T, w[i], [&](int k, int n, double2 xk, double2 xn) {
				X[k] = xk; X[n] = xn;
				buf[spad(k)] = xk; buf[spad(n)] = xn;
			});
		// (2) S = X_j H_0 + sum_{p>=1} X_{j-p} H_p (+ Y_j) for the owned bins, one row (pair) at a time for all eight
		//     bin pairs: 16 independent 16-byte loads in flight per pass instead of whatever fits next to the sums of
		//     one bin pair -- the phase is a chain of memory round trips, nothing else.  The running sum is parked in
		//     the buffer, in place of X_j (which is in the FDL by now).  Rows that are read once go past the L1
		//     (__ldcg): the kernel lives on what the two resident CTAs' buffers leave of it (twiddle tables, a
		//     shared filter).  Then the inverse merge.
#define L0_K(i) (t + (i) * T)
#define L0_N(i) ((L0_K(i) == 0) ? N / 2 : N - L0_K(i))
		{
			double2 hk[8], hn[8];
#pragma unroll
			for (int i = 0; i < 8; ++i) {
				hk[i] = per_ch_h ? __ldcg(&H[L0_K(i)]) : H[L0_K(i)];
				hn[i] = per_ch_h ? __ldcg(&H[L0_N(i)]) : H[L0_N(i)];
			}
#pragma unroll
			for (int i = 0; i < 8; ++i) {
				const int k = L0_K(i), n = L0_N(i);
				const double2 xk = buf[spad(k)], xn = buf[spad(n)];
				buf[spad(k)] = (k == 0) ? make_double2(xk.x * hk[i].x, xk.y * hk[i].y) : cmul(xk, hk[i]);   // packed bin: two real products
				buf[spad(n)] = cmul(xn, hn[i]);
			}
		}
		auto mac_partition = [&](int p) {
			const double2 *Xp = fdl + (long) ring_back(a.slot, p, a.fdl_rows) * N, *Hp = H + (long) p * N;
#pragma unroll
			for (int half = 0; half < 8; half += 4) {
				double2 xk[4], xn[4], hk[4], hn[4];
#pragma unroll
				for (int i = 0; i < 4; ++i) {
					const int k = L0_K(half + i), n = L0_N(half + i);
					xk[i] = __ldcg(&Xp[k]);
					xn[i] = __ldcg(&Xp[n]);
					hk[i] = per_ch_h ? __ldcg(&Hp[k]) : Hp[k];
					hn[i] = per_ch_h ? __ldcg(&Hp[n]) : Hp[n];
				}
#pragma unroll
				for (int i = 0; i < 4; ++i) {
					const int k = L0_K(half + i), n = L0_N(half + i);
					double2 Sk = buf[spad(k)];
					cmac_packed(Sk, xk[i], hk[i], k == 0);
					buf[spad(k)] = Sk;
					buf[spad(n)] = cmac(buf[spad(n)], xn[i], hn[i]);
				}
			}
		};
		if constexpr (P > 0) {
#pragma unroll
			for (int p = 1; p < P; ++p) mac_partition(p);
		}
		else {
			// (the two transform groups of a 2048-point CTA may loop a different number of times: no barrier inside)
			const int np = (a.cls_T > 0) ? fir_fused_parts(a.blk, s, a.cls_T, a.cls_K, a.cls_w, a.la, a.pass_m, a.P) : a.P;
#pragma unroll 1
			for (int p = 1; p < np; ++p) mac_partition(p);
		}
#pragma unroll
		for (int half = 0; half < 8; half += 4) {
			// what the other partitions of this level contribute (`init`: Y_j of the per-block MAC, or the batch tier's
			// V_j when this kernel sums the near partitions itself): summed here, in the frequency domain, so that the
			// level needs one inverse transform
			double2 yk[4], yn[4], w2[4];
#pragma unroll
			for (int i = 0; i < 4; ++i) {
				w2[i] = __ldg(&a.tw[L0_K(half + i)]);
				if (init) {
					yk[i] = __ldcg(&init[L0_K(half + i)]);
					yn[i] = __ldcg(&init[L0_N(half + i)]);
				}
			}
#pragma unroll
			for (int i = 0; i < 4; ++i) {
				const int k = L0_K(half + i), n = L0_N(half + i);
				double2 Sk = buf[spad(k)], Sn = buf[spad(n)];
				if (init) {
					Sk = cadd(Sk, yk[i]);
					Sn = cadd(Sn, yn[i]);
				}
				irfft_merge<N>(buf, k, n, Sk, Sn, w2[i]);
			}
		}
#undef L0_K
#undef L0_N
	}
	__syncthreads();
	fft_forward_smem<N>(buf, a.ptw, t);
	if (active) {
		const double scale = 1.0 / N;
		double2 *carry = reinterpret_cast<double2 *>(a.carry + (long) s * N);
		double2 *out = reinterpret_cast<double2 *>(a.out + (long) s * a.out_ch_stride);
		double *yc = a.yout ? a.yout + (a.yout_map ? a.yout_map[s] : s) : nullptr;
		double2 c[8];
#pragma unroll
		for (int i = 0; i < 8; ++i) c[i] = __ldcg(&carry[t + i * T]);
#pragma unroll
		for (int i = 0; i < 8; ++i) {
			const int n = t + i * T;
			const double2 lo = buf[spad(n)], hi = buf[spad(n + N / 2)];
			const double2 y = ola_out(lo, scale, c[i]);
			if (CL) {
				buf[spad(n)] = y;   // this thread is the only one that touches entry n after the last pass
				if (FIR_L0_ASYNC) carry[n] = ola_scaled(hi, scale);
			}
			else if (yc) {
				yc[2L * n * a.yout_stride] = y.x;
				yc[(2L * n + 1) * a.yout_stride] = y.y;
			}
			else out[n] = y;
			// (cluster form with fenced barriers: the new carry is stored after the barrier below -- its release fence
			// would wait for these stores; the second half of the buffer, where it comes from, is nobody else's)
			if (!CL) carry[n] = ola_scaled(hi, scale);
		}
	}
	if constexpr (CL) {
		const int s0 = ((int) blockIdx.x - (int) crank) * CPB;
		double *yr = a.yout + (a.yout_map ? a.yout_map[s0] : s0);
#if FIR_L0_ASYNC
		// every thread of the cluster has read its second half (the carry stores above depend on those loads): the
		// second halves are free to receive
		fence_proxy_async_smem();
		cluster_barrier_relaxed();
		if (threadIdx.x == 0) {
			// rows [wr * NPC, (wr + 1) * NPC) of every channel of this CTA go to CTA wr, which writes them
			const uint32_t mb = smem_u32(&mbar[1]);
#pragma unroll
			for (int wr = 0; wr < NCL; ++wr) {
#pragma unroll
				for (int gg = 0; gg < CPB; ++gg) {
					const int cc = (int) crank * CPB + gg;   // this channel within the cluster's four
					bulk_s2c(mapa_u32(smem_u32(stage(cc)), wr), smem_u32(smem + (size_t) gg * FftCfg<N>::STRIDE + spad(wr * NPC)),
					         CHUNK_BYTES, mapa_u32(mb, wr));
				}
			}
		}
		mbar_wait_cluster(&mbar[1], 0);   // this CTA's rows of all four channels have landed in `stage`
#pragma unroll
		for (int i = 0; i < NPC / THREADS; ++i) {
			const int n = (int) crank * NPC + (int) threadIdx.x + i * THREADS, nl = spad((int) threadIdx.x + i * THREADS);
			const double2 y0 = stage(0)[nl], y1 = stage(1)[nl], y2 = stage(2)[nl], y3 = stage(3)[nl];
			double *r0 = yr + 2L * n * a.yout_stride, *r1 = r0 + a.yout_stride;
			*reinterpret_cast<double2 *>(r0) = make_double2(y0.x, y1.x);
			*reinterpret_cast<double2 *>(r0 + 2) = make_double2(y2.x, y3.x);
			*reinterpret_cast<double2 *>(r1) = make_double2(y0.y, y1.y);
			*reinterpret_cast<double2 *>(r1 + 2) = make_double2(y2.y, y3.y);
		}
		cluster_barrier_relaxed();   // nobody leaves before the copies out of its shared memory are complete (execution only)
#else
		cg::cluster_group cluster = cg::this_cluster();
		cluster.sync();   // all four channels' results are in their owners' buffers
#pragma unroll
		for (int i = 0; i < NPC / THREADS; ++i) {
			const int n = (int) crank * NPC + (int) threadIdx.x + i * THREADS;
			const double2 y0 = rbuf[0][spad(n)], y1 = rbuf[1][spad(n)], y2 = rbuf[2][spad(n)], y3 = rbuf[3][spad(n)];
			double *r0 = yr + 2L * n * a.yout_stride, *r1 = r0 + a.yout_stride;
			*reinterpret_cast<double2 *>(r0) = make_double2(y0.x, y1.x);
			*reinterpret_cast<double2 *>(r0 + 2) = make_double2(y2.x, y3.x);
			*reinterpret_cast<double2 *>(r1) = make_double2(y0.y, y1.y);
			*reinterpret_cast<double2 *>(r1 + 2) = make_double2(y2.y, y3.y);
		}
		{
			const double scale = 1.0 / N;
			double2 *carry = reinterpret_cast<double2 *>(a.carry + (long) s * N);
#pragma unroll
			for (int i = 0; i < 8; ++i) carry[t + i * T] = ola_scaled(buf[spad(t + i * T + N / 2)], scale);
		}
		cluster_barrier_relaxed();   // nobody leaves while its buffer may still be read (execution only: nothing to publish)
#endif
	}
}

// dspb200_debug_stall(): one thread waits `ns` nanoseconds of %globaltimer (at most FIR_STALL_MAX_US) and ends; the
// iteration cap bounds the loop whatever the timer does
__global__ void k_fir_stall(long long ns)
{
	unsigned long long t0, t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
	for (int i = 0; i < (1 << 18); ++i) {
		asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
		if ((long long) (t - t0) >= ns) break;
		__nanosleep(256);
	}
}

// Y[s][k] = sum_{p in [p0,p1)} FDL[s][(slot0 - p) mod P][k] * H[s or 0][p][k]   (packed bin 0)
// The HBM-streaming kernel of the engine: 32 bytes in per complex MAC (16 with a shared IR, whose
// rows stay in L2), 4 DFMA.
struct MacArgs {
	const double2 *fdl;   // [s][P][N]
	const double2 *H;     // [s][P][N] or [P][N]
	double2 *Y;           // [s][N]
	const double2 *init;  // [s][N] spectrum to start from (NULL: zero)
	int N, P;
	int slot0, p0, p1;
	long h_ch_stride;     // P*N or 0 (shared IR)
};

#ifndef FIR_MAC_MINB
#define FIR_MAC_MINB 3
#endif
// Bin 0 of a row is packed (DC and Nyquist, both real: two real products instead of a complex one).  Only the warp
// that holds it compiles the special case (DCW); everywhere else the inner loop is the plain complex MAC, without
// predicated-off copies of every FMA.
template <bool SHARED_H, bool DCW>
__device__ __forceinline__ void fir_mac_body(const MacArgs &a, int y)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	const int s = y;
	const double2 *fdl = a.fdl + (long) s * a.P * a.N + k;
	const double2 *H = a.H + (long) s * a.h_ch_stride + k;
	double2 acc0 = a.init ? __ldcs(&a.init[(long) s * a.N + k]) : make_double2(0.0, 0.0);
	double2 acc1 = make_double2(0.0, 0.0), acc2 = acc1, acc3 = acc1;
	const bool dc = DCW && (k == 0);
	int slot = a.slot0 - a.p0;
	slot %= a.P;
	if (slot < 0) slot += a.P;
	int p = a.p0;

#define LOAD_X(q) __ldcs(&fdl[(long) ((slot - (q) < 0) ? slot - (q) + a.P : slot - (q)) * a.N])
#define LOAD_H(q) (SHARED_H ? __ldg(&H[(long) (p + (q)) * a.N]) : __ldcs(&H[(long) (p + (q)) * a.N]))
#define CMAC(ACC, XV, HV)                                            \
	do {                                                             \
		if (dc) {                                                    \
			ACC.x = fma(XV.x, HV.x, ACC.x);                          \
			ACC.y = fma(XV.y, HV.y, ACC.y);                          \
		}                                                            \
		else {                                                       \
			ACC.x = fma(XV.x, HV.x, fma(-XV.y, HV.y, ACC.x));        \
			ACC.y = fma(XV.x, HV.y, fma(XV.y, HV.x, ACC.y));         \
		}                                                            \
	} while (0)

	for (; p + 4 <= a.p1; p += 4) {
		const double2 x0 = LOAD_X(0), x1 = LOAD_X(1), x2 = LOAD_X(2), x3 = LOAD_X(3);
		const double2 h0 = LOAD_H(0), h1 = LOAD_H(1), h2 = LOAD_H(2), h3 = LOAD_H(3);
		CMAC(acc0, x0, h0);
		CMAC(acc1, x1, h1);
		CMAC(acc2, x2, h2);
		CMAC(acc3, x3, h3);
		slot -= 4;
		if (slot < 0) slot += a.P;
	}
	for (; p < a.p1; ++p) {
		const double2 x0 = LOAD_X(0);
		const double2 h0 = LOAD_H(0);
		CMAC(acc0, x0, h0);
		slot -= 1;
		if (slot < 0) slot += a.P;
	}
#undef LOAD_X
#undef LOAD_H
#undef CMAC
	a.Y[(long) s * a.N + k] = make_double2((acc0.x + acc1.x) + (acc2.x + acc3.x), (acc0.y + acc1.y) + (acc2.y + acc3.y));
}

template <bool SHARED_H>
__global__ void __launch_bounds__(256, FIR_MAC_MINB) k_fir_mac(MacArgs a)
{
	if (blockIdx.x == 0 && threadIdx.x < 32) fir_mac_body<SHARED_H, true>(a, blockIdx.y);
	else fir_mac_body<SHARED_H, false>(a, blockIdx.y);
}

// Time-batched tail of the last level.  One launch after block q completes produces V_j for the T periods
// j = q+pf+1 .. q+pf+T at once (pf = partitions summed inside the fused FFT kernel): every FDL row and every filter
// row is streamed ONCE for T outputs (the filter rows slide through a T-deep register window), instead of once per
// output.  Which partitions a period gets: fir_batch_window() (fir_plan.h).  Tiers: a deeper batch (larger T) reads the
// filter less often; the far tier's result is the near tier's starting value `Vin`.
struct MacBatchArgs {
	const double2 *fdl;   // [s][P][N]
	const double2 *H;     // [s][P][N] or [P][N]
	double2 *V;           // [slot][s][N], slot = j mod n_slots
	int N, P, n_sel;      // P: rows of the FDL ring = partitions of the level
	long q;               // block that just completed
	int n_slots;
	long h_ch_stride;
	// a FirTierLaunch (fir_plan.h): blockIdx.y = y < n_tier_y is row y of class g, the rest the pass rows of class pass_g
	int pf;
	int g, K, w;
	int p_lo, p_hi;
	const double2 *Vin;   // [slot][s][N], slot = j mod vin_slots: a farther tier's sums to start from (NULL: zero)
	int vin_slots;
	int n_tier_y, pass_g, pass_m;
};

#ifndef FIR_BATCH_PREFETCH
#define FIR_BATCH_PREFETCH 0
#endif
template <int T>
struct MacBatchCfg {
#if FIR_BATCH_PREFETCH
	// software-pipelined form: eight more 16-byte registers per thread (the next four rows of X and H in flight)
	static constexpr int THREADS = (T <= 4) ? 256 : 128;
	static constexpr int MINB = (T <= 4) ? 2 : (T <= 8) ? 3 : 2;
#else
	static constexpr int THREADS = (T <= 8) ? 256 : 128;
	static constexpr int MINB = (T <= 4) ? FIR_MAC_MINB : (T <= 8) ? 2 : (T <= 12) ? 3 : 2;
#endif
};

// PASS: the mid-window pass role, V read and written in place by the thread that owns the element
template <int T, bool SHARED_H, bool DCW, bool PASS = false>
__device__ __forceinline__ void fir_mac_batch_body(const MacBatchArgs &a, int y)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	const int s = fir_class_channel(PASS ? a.pass_g : a.g, a.K, a.w, y);
	const FirBatchWindow win = fir_batch_window(PASS, T, a.p_lo, a.p_hi, a.pass_m);
	const int x_hi = win.x_hi, h_hi = win.h_hi, n_t = win.n_t;
	const double2 *Vin = PASS ? a.V : a.Vin;
	const int vin_slots = PASS ? a.n_slots : a.vin_slots;
	const double2 *fdl = a.fdl + (long) s * a.P * a.N + k;
	const double2 *H = a.H + (long) s * a.h_ch_stride + k;
	const bool dc = DCW && (k == 0);
	const double2 zero = make_double2(0.0, 0.0);
	double2 acc[T], hw[T];
	// bit t of `live`: hw[t] is a filter row of period t's window (the NaN rule: window_mac())
#define HLIVE(p) ((p) >= a.p_lo && (p) < h_hi)
#define HROW(p) (HLIVE(p) ? (SHARED_H ? __ldg(&H[(long) (p) * a.N]) : __ldcs(&H[(long) (p) * a.N])) : zero)
	int m = a.pf + 1;   // first row: the newest complete block, X_q
	unsigned live = 0;
#pragma unroll
	for (int t = 0; t < T; ++t) {
		const long j = a.q + a.pf + 1 + t;
		acc[t] = (Vin && t < n_t) ? __ldcs(&Vin[((j % vin_slots) * a.n_sel + s) * (long) a.N + k]) : zero;
		hw[t] = HROW(m + t);
		live |= (unsigned) HLIVE(m + t) << t;
	}
	int slot = (int) (a.q % a.P);   // row of X_{q+pf+1-m} = X_q
#define XROW(d) __ldcs(&fdl[(long) ((slot - (d) < 0) ? slot - (d) + a.P : slot - (d)) * a.N])
#define STEP(XV, HN, PN)                                                      \
	do {                                                                      \
		window_mac<T>(acc, hw, live, XV, dc);                                 \
		_Pragma("unroll") for (int t = 0; t + 1 < T; ++t) hw[t] = hw[t + 1];  \
		hw[T - 1] = HN;                                                       \
		live = (live >> 1) | ((unsigned) HLIVE(PN) << (T - 1));               \
	} while (0)
#if FIR_BATCH_PREFETCH
	// the eight loads of the NEXT four rows are issued before the current four are used; rows past the tier are zeros
#define XROWG(mm, d) (((mm) + (d) < x_hi) ? XROW(d) : zero)
	double2 x0 = XROWG(m, 0), x1 = XROWG(m, 1), x2 = XROWG(m, 2), x3 = XROWG(m, 3);
	double2 h0 = HROW(m + T), h1 = HROW(m + T + 1), h2 = HROW(m + T + 2), h3 = HROW(m + T + 3);
	for (; m < x_hi; m += 4) {
		slot -= 4;
		if (slot < 0) slot += a.P;
		const int mn = m + 4;
		const double2 nx0 = XROWG(mn, 0), nx1 = XROWG(mn, 1), nx2 = XROWG(mn, 2), nx3 = XROWG(mn, 3);
		const double2 nh0 = HROW(mn + T), nh1 = HROW(mn + T + 1), nh2 = HROW(mn + T + 2), nh3 = HROW(mn + T + 3);
		STEP(x0, h0, m + T);
		STEP(x1, h1, m + T + 1);
		STEP(x2, h2, m + T + 2);
		STEP(x3, h3, m + T + 3);
		x0 = nx0; x1 = nx1; x2 = nx2; x3 = nx3;
		h0 = nh0; h1 = nh1; h2 = nh2; h3 = nh3;
	}
#undef XROWG
#else
	for (; m + 4 <= x_hi; m += 4) {
		// eight independent 16-byte loads in flight per thread, as in k_fir_mac
		const double2 x0 = XROW(0), x1 = XROW(1), x2 = XROW(2), x3 = XROW(3);
		const double2 h0 = HROW(m + T), h1 = HROW(m + T + 1), h2 = HROW(m + T + 2), h3 = HROW(m + T + 3);
		STEP(x0, h0, m + T);
		STEP(x1, h1, m + T + 1);
		STEP(x2, h2, m + T + 2);
		STEP(x3, h3, m + T + 3);
		slot -= 4;
		if (slot < 0) slot += a.P;
	}
	for (; m < x_hi; ++m) {
		const double2 x0 = XROW(0);
		const double2 h0 = HROW(m + T);
		STEP(x0, h0, m + T);
		slot = (slot == 0) ? a.P - 1 : slot - 1;
	}
#endif
#undef XROW
#undef STEP
#undef HROW
#undef HLIVE
#pragma unroll
	for (int t = 0; t < T; ++t) {
		const long j = a.q + a.pf + 1 + t;
		if (t < n_t) a.V[((j % a.n_slots) * a.n_sel + s) * (long) a.N + k] = acc[t];
	}
}

template <int T, bool SHARED_H>
__global__ void __launch_bounds__(MacBatchCfg<T>::THREADS, MacBatchCfg<T>::MINB) k_fir_mac_batch(MacBatchArgs a)
{
	const bool dcw = blockIdx.x == 0 && threadIdx.x < 32;   // the warp that holds the packed bin 0
	if (a.pass_m > 0 && (int) blockIdx.y >= a.n_tier_y) {
		if (dcw) fir_mac_batch_body<T, SHARED_H, true, true>(a, (int) blockIdx.y - a.n_tier_y);
		else fir_mac_batch_body<T, SHARED_H, false, true>(a, (int) blockIdx.y - a.n_tier_y);
	}
	else if (dcw) fir_mac_batch_body<T, SHARED_H, true>(a, blockIdx.y);
	else fir_mac_batch_body<T, SHARED_H, false>(a, blockIdx.y);
}

// The per-block MAC and the staggered batch launch of the same block period in ONE grid: rows [0, n_batch_y) of the grid
// are the batch tier's channels of this block's residue class (long CTAs first), the rest the per-block MAC of every
// channel.  Neither depends on the other (both read blocks <= q and what earlier launches produced), and together
// they fill the machine evenly: alone, a class launch of the batch tier is a few waves of long CTAs and the MAC a short
// kernel with its own ramps.
struct TailArgs {
	MacArgs m;
	MacBatchArgs b;
	int n_batch_y;
};

template <int T, bool SHARED_H>
__global__ void __launch_bounds__(256, FIR_MAC_MINB) k_fir_tail(TailArgs a)
{
	const bool dcw = blockIdx.x == 0 && threadIdx.x < 32;
	if ((int) blockIdx.y < a.n_batch_y) {
		if (dcw) fir_mac_batch_body<T, SHARED_H, true>(a.b, blockIdx.y);
		else fir_mac_batch_body<T, SHARED_H, false>(a.b, blockIdx.y);
	}
	else {
		if (dcw) fir_mac_body<SHARED_H, true>(a.m, (int) blockIdx.y - a.n_batch_y);
		else fir_mac_body<SHARED_H, false>(a.m, (int) blockIdx.y - a.n_batch_y);
	}
}

static int batch_threads_for(int T)
{
	return (T == 16) ? MacBatchCfg<16>::THREADS : (T == 12) ? MacBatchCfg<12>::THREADS : (T == 8) ? MacBatchCfg<8>::THREADS
	     : (T == 6) ? MacBatchCfg<6>::THREADS : MacBatchCfg<4>::THREADS;
}

// `smem`: dynamic shared memory the kernel does not use -- a cap on its CTAs per SM (a whole-launch far tier otherwise
// fills every SM's registers with long-lived CTAs, and the next block's fused kernel waits for them to retire)
template <int T>
static void launch_mac_batch_t(bool shared_h, dim3 grid, int threads, cudaStream_t st, const MacBatchArgs &b, size_t smem)
{
	if (smem > 48 * 1024) {
		static std::atomic<size_t> set[64];
		int dev = 0;
		cudaGetDevice(&dev);
		if (set[dev & 63].load() < smem) {
			cudaFuncSetAttribute((k_fir_mac_batch<T, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
			cudaFuncSetAttribute((k_fir_mac_batch<T, false>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem);
			set[dev & 63].store(smem);
		}
	}
	if (shared_h) LAUNCH((k_fir_mac_batch<T, true>), grid, threads, smem, st, b);
	else LAUNCH((k_fir_mac_batch<T, false>), grid, threads, smem, st, b);
}

// grid: x = N / threads, y = channels of this launch; `threads` at most batch_threads_for(T)
static void launch_mac_batch(int T, bool shared_h, dim3 grid, int threads, cudaStream_t st, const MacBatchArgs &b, const char *prof_name = "fir_mac_batch",
                             size_t smem = 0)
{
	ProfScope prof(prof_name, st);
	switch (T) {
	case 16: launch_mac_batch_t<16>(shared_h, grid, threads, st, b, smem); break;
	case 12: launch_mac_batch_t<12>(shared_h, grid, threads, st, b, smem); break;
	case 8: launch_mac_batch_t<8>(shared_h, grid, threads, st, b, smem); break;
	case 6: launch_mac_batch_t<6>(shared_h, grid, threads, st, b, smem); break;
	default: launch_mac_batch_t<4>(shared_h, grid, threads, st, b, smem); break;
	}
}

// Bulk form of the whole convolution sum for calls that bring several whole blocks at once (offline rendering,
// `dsp -b 65536`): Y_i = sum_{p<P} X_{j+i-p} H_p for the nb <= T new blocks i in ONE pass -- every FDL row
// (P + T - 1 of them) and every filter row is streamed once for T outputs, the filter rows slide through a
// T-deep register window.  Outputs i >= nb are computed on rows that do not exist yet and dropped.

struct MacBulkArgs {
	const double2 *fdl;   // [s][rows][N]
	const double2 *H;     // [s][P][N] or [P][N]
	double2 *Y;           // [i][s][N]
	int N, P, rows, n_sel, nb;
	long j;               // first new block (its spectrum is in row j % rows)
	long h_ch_stride;
};

template <int T, bool SHARED_H>
__global__ void __launch_bounds__(256) k_fir_mac_bulk(MacBulkArgs a)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	const int s = blockIdx.y;
	const double2 *fdl = a.fdl + (long) s * a.rows * a.N + k;
	const double2 *H = a.H + (long) s * a.h_ch_stride + k;
	const bool dc = (k == 0);
	const double2 zero = make_double2(0.0, 0.0);
	double2 acc[T], hw[T];
	// bit i of `live`: hw[i] is a filter row (0 <= d + i < P); the NaN rule (window_mac()) keeps a NaN or Inf in the row
	// of a later block of this call (or a stale row past the new ones) out of the outputs of earlier blocks
#define HLIVE(p) ((p) >= 0 && (p) < a.P)
#define HROW(p) (HLIVE(p) ? (SHARED_H ? __ldg(&H[(long) (p) * a.N]) : __ldcs(&H[(long) (p) * a.N])) : zero)
	// step d = P-1 .. -(T-1): block m = j - d meets H_{d+i} for output i; window hw[i] = H_{d+i}
	int d = a.P - 1;
	unsigned live = 0;
#pragma unroll
	for (int i = 0; i < T; ++i) {
		acc[i] = zero;
		hw[i] = HROW(d + i);
		live |= (unsigned) HLIVE(d + i) << i;
	}
	int slot = (int) (((a.j - d) % a.rows + a.rows) % a.rows);   // row of X_{j-d}; grows by one per step
#define XROW(e) __ldcs(&fdl[(long) ((slot + (e) >= a.rows) ? slot + (e) - a.rows : slot + (e)) * a.N])
#define STEP(XV, HN, PN)                                                      \
	do {                                                                      \
		window_mac<T>(acc, hw, live, XV, dc);                                 \
		_Pragma("unroll") for (int i = T - 1; i > 0; --i) hw[i] = hw[i - 1];  \
		hw[0] = HN;                                                           \
		live = ((live << 1) | (unsigned) HLIVE(PN)) & ((1u << T) - 1);        \
	} while (0)
	const int steps = a.P + T - 1;
	int n = 0;
	for (; n + 4 <= steps; n += 4) {
		const double2 x0 = XROW(0), x1 = XROW(1), x2 = XROW(2), x3 = XROW(3);
		const double2 h0 = HROW(d - 1), h1 = HROW(d - 2), h2 = HROW(d - 3), h3 = HROW(d - 4);
		STEP(x0, h0, d - 1);
		STEP(x1, h1, d - 2);
		STEP(x2, h2, d - 3);
		STEP(x3, h3, d - 4);
		d -= 4;
		slot += 4;
		if (slot >= a.rows) slot -= a.rows;
	}
	for (; n < steps; ++n) {
		const double2 x0 = XROW(0);
		const double2 h0 = HROW(d - 1);
		STEP(x0, h0, d - 1);
		d -= 1;
		slot = (slot + 1 == a.rows) ? 0 : slot + 1;
	}
#undef XROW
#undef STEP
#undef HROW
#undef HLIVE
#pragma unroll
	for (int i = 0; i < T; ++i)
		if (i < a.nb) a.Y[((long) i * a.n_sel + s) * a.N + k] = acc[i];
}

// bulk overlap-add + transpose: frame i B + f of the call = lo[i][s][f] + (i == 0 ? carry[s][f] : hi[i-1][s][f])
__global__ void __launch_bounds__(256) k_fir_unstash_bulk(const double *__restrict__ lo, const double *__restrict__ hi, const double *__restrict__ carry,
                                                          int B, double *__restrict__ out, long stride, const int *__restrict__ ch_map, int n_sel)
{
	__shared__ double tile[32][33];
	const int f0 = blockIdx.x * 32, s0 = blockIdx.y * 32, i = blockIdx.z;
	const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
	const double *prev = (i == 0) ? carry : hi + (long) (i - 1) * n_sel * B;
	const double *cur = lo + (long) i * n_sel * B;
#pragma unroll
	for (int r = ty; r < 32; r += 8) {
		const int s = s0 + r, f = f0 + tx;
		tile[r][tx] = (s < n_sel && f < B) ? cur[(long) s * B + f] + prev[(long) s * B + f] : 0.0;
	}
	__syncthreads();
	double *o = out + (long) i * B * stride;
#pragma unroll
	for (int r = ty; r < 32; r += 8) {
		const int f = f0 + r, s = s0 + tx;
		if (f < B && s < n_sel) o[(long) f * stride + (ch_map ? ch_map[s] : s)] = tile[tx][r];
	}
}

// general path: out[m] = pre[m] + pend(m) + sum_{r<=m} x[r] h0[m-r], m = pos+i; x = current level-0 block in the ring
__global__ void k_fir_head(const double *hist, long hist_len, long blk_off, const double *pre, const double *h0, long h0_ch_stride,
                           PendArgs pend, double *out, long stride, const int *ch_map, int B, int pos, int seg)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	const int s = blockIdx.y;
	if (i >= seg) return;
	const int m = pos + i;
	const double *x = hist + (long) s * hist_len + blk_off;
	const double *h = h0 + (long) s * h0_ch_stride;
	double acc0 = pre[(long) s * B + m], acc1 = 0.0;
	for (int l = 0; l < pend.n; ++l) acc1 += pend.buf[l][(long) s * pend.len[l] + pend.off[l] + i];
	int r = 0;
	for (; r + 2 <= m + 1; r += 2) {
		acc0 = fma(x[r], h[m - r], acc0);
		acc1 = fma(x[r + 1], h[m - r - 1], acc1);
	}
	if (r <= m) acc0 = fma(x[r], h[m - r], acc0);
	out[(long) i * stride + (ch_map ? ch_map[s] : s)] = acc0 + acc1;
}

// fir.c latency: out[a] = y[a - L]; ring slot of absolute frame a is a % L
__global__ void k_delay_read(const double *y, long y_stride, const double *ring, double *out, long stride,
                             const int *ch_map, int n_sel, long frames, long L, long abs0)
{
	const long idx = (long) blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= frames * n_sel) return;
	const long i = idx / n_sel;
	const int s = (int) (idx - i * n_sel);
	const double v = (i < L) ? ring[((abs0 + i) % L) * n_sel + s] : y[(i - L) * y_stride + s];
	out[i * stride + ch_map[s]] = v;
}

__global__ void k_delay_write(const double *y, long y_stride, double *ring, int n_sel, long frames, long L, long abs0)
{
	const long idx = (long) blockIdx.x * blockDim.x + threadIdx.x;
	const long first = (frames > L) ? frames - L : 0;
	const long cnt = frames - first;
	if (idx >= cnt * n_sel) return;
	const long i = first + idx / n_sel;
	const int s = (int) (idx % n_sel);
	ring[((abs0 + i) % L) * n_sel + s] = y[i * y_stride + s];
}

// ------------------------------------------------------------------------------------------
// launch helpers (dispatch on the FFT size)
// ------------------------------------------------------------------------------------------
// Dynamic shared memory of the fused block kernel: what the transform buffers need, or more on request
// (DSP_B200_FIR_L0_SMEM_KB: a way to cap its CTAs per SM, so that the streaming kernels of the other streams find
// registers next to it)
template <int N>
static size_t level0_smem(bool cluster_form = false)
{
	static const long want = getenv("DSP_B200_FIR_L0_SMEM_KB") ? atol(getenv("DSP_B200_FIR_L0_SMEM_KB")) * 1024 : 0;
	size_t n = cluster_form ? L0ClCfg<N>::SMEM : FftCfg<N>::SMEM;
	if (N >= 2048 && want > (long) n) n = (size_t) ((want > 227 * 1024) ? 227 * 1024 : want);
	return n;
}

template <int N>
static int configure_n()
{
	static std::atomic<int> configured[64];
	int dev = 0;
	cudaGetDevice(&dev);
	if (!configured[dev & 63].load()) {
		CUDA_TRY(cudaFuncSetAttribute(k_fir_fwd<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) FftCfg<N>::SMEM), return -1);
		CUDA_TRY(cudaFuncSetAttribute(k_fir_inv<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) FftCfg<N>::SMEM), return -1);
		CUDA_TRY(cudaFuncSetAttribute((k_fir_level0<N, 1>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int) level0_smem<N>()), return -1);
		CUDA_TRY(cudaFuncSetAttribute((k_fir_level0<N, 2>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int) level0_smem<N>()), return -1);
		CUDA_TRY(cudaFuncSetAttribute((k_fir_level0<N, 0>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int) level0_smem<N>()), return -1);
		if constexpr (FftCfg<N>::CPB <= 2) {
			CUDA_TRY(cudaFuncSetAttribute((k_fir_level0<N, 1, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int) level0_smem<N>(true)), return -1);
			CUDA_TRY(cudaFuncSetAttribute((k_fir_level0<N, 2, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int) level0_smem<N>(true)), return -1);
			CUDA_TRY(cudaFuncSetAttribute((k_fir_level0<N, 0, true>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int) level0_smem<N>(true)), return -1);
		}
		configured[dev & 63].store(1);
	}
	return 0;
}

template <int N>
static int launch_fwd_n(const FwdArgs &a, cudaStream_t st, int nb)
{
	if (configure_n<N>()) return -1;
	if (a.n_ch <= 0) return 0;
	ProfScope prof("fir_fwd", st);
	LAUNCH(k_fir_fwd<N>, dim3(ceil_div(a.n_ch, FftCfg<N>::CPB), nb), FftCfg<N>::THREADS, FftCfg<N>::SMEM, st, a);
	return 0;
}

template <int N>
static int launch_inv_n(const InvArgs &a, cudaStream_t st, int nb)
{
	if (configure_n<N>()) return -1;
	if (a.n_ch <= 0) return 0;
	ProfScope prof("fir_inv", st);
	LAUNCH(k_fir_inv<N>, dim3(ceil_div(a.n_ch, FftCfg<N>::CPB), nb), FftCfg<N>::THREADS, FftCfg<N>::SMEM, st, a);
	return 0;
}

template <int N>
static int launch_level0_n(const L0Args &a, cudaStream_t st)
{
	if (configure_n<N>()) return -1;
	if (a.n_ch <= 0) return 0;
	ProfScope prof("fir_level0", st);
	if constexpr (FftCfg<N>::CPB <= 2) {
		if (a.cluster_io) {
			constexpr int CPB = FftCfg<N>::CPB;
			cudaLaunchConfig_t cfg = {};
			cfg.gridDim = dim3(a.n_ch / CPB); cfg.blockDim = dim3(FftCfg<N>::THREADS); cfg.dynamicSmemBytes = level0_smem<N>(true); cfg.stream = st;
			cudaLaunchAttribute attr;
			attr.id = cudaLaunchAttributeClusterDimension;
			attr.val.clusterDim.x = 4 / CPB; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
			cfg.attrs = &attr; cfg.numAttrs = 1;
			if (a.P == 1) CUDA_TRY(cudaLaunchKernelEx(&cfg, k_fir_level0<N, 1, true>, a), return -1);
			else if (a.P == 2) CUDA_TRY(cudaLaunchKernelEx(&cfg, k_fir_level0<N, 2, true>, a), return -1);
			else CUDA_TRY(cudaLaunchKernelEx(&cfg, k_fir_level0<N, 0, true>, a), return -1);
			g_kernel_launches.fetch_add(1, std::memory_order_relaxed);
			return 0;
		}
	}
	if (a.P == 1) LAUNCH((k_fir_level0<N, 1>), ceil_div(a.n_ch, FftCfg<N>::CPB), FftCfg<N>::THREADS, level0_smem<N>(), st, a);
	else if (a.P == 2) LAUNCH((k_fir_level0<N, 2>), ceil_div(a.n_ch, FftCfg<N>::CPB), FftCfg<N>::THREADS, level0_smem<N>(), st, a);
	else LAUNCH((k_fir_level0<N, 0>), ceil_div(a.n_ch, FftCfg<N>::CPB), FftCfg<N>::THREADS, level0_smem<N>(), st, a);
	return 0;
}

// the persistent pipeline (fir_pipe.cuh): one CTA per SM, channels strided over the grid
template <int N>
static int launch_pipe_n(const PipeArgs &a, cudaStream_t st)
{
	static std::atomic<int> configured[64];
	int dev = 0;
	cudaGetDevice(&dev);
	if (!configured[dev & 63].load()) {
		CUDA_TRY(cudaFuncSetAttribute(k_fir_pipe<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) PipeCfg<N>::SMEM), return -1);
		configured[dev & 63].store(1);
	}
	if (a.n_ch <= 0) return 0;
	int grid = sm_count();
	if (grid < 1) return -1;
	if (const char *e = getenv("DSP_B200_FIR_PIPE_GRID")) grid = atoi(e);
	if (grid > a.n_ch) grid = a.n_ch;
	if (grid < 1) grid = 1;
	ProfScope prof("fir_pipe", st);
	LAUNCH(k_fir_pipe<N>, grid, PipeCfg<N>::THREADS, PipeCfg<N>::SMEM, st, a);
	return 0;
}

static int launch_pipe(int N, const PipeArgs &a, cudaStream_t st)
{
	switch (N) {
	case 2048: return launch_pipe_n<2048>(a, st);
	case 4096: return launch_pipe_n<4096>(a, st);
	default: set_error("pipeline kernel: unsupported block size %d", N); return -1;
	}
}

#define DISPATCH_N(N_, FN, ...)                      \
	switch (N_) {                                    \
	case 64: return FN<64>(__VA_ARGS__);             \
	case 128: return FN<128>(__VA_ARGS__);           \
	case 256: return FN<256>(__VA_ARGS__);           \
	case 512: return FN<512>(__VA_ARGS__);           \
	case 1024: return FN<1024>(__VA_ARGS__);         \
	case 2048: return FN<2048>(__VA_ARGS__);         \
	case 4096: return FN<4096>(__VA_ARGS__);         \
	case 8192: return FN<8192>(__VA_ARGS__);         \
	default: set_error("unsupported FFT size %d", N_); return -1; \
	}

static int launch_fwd(int N, const FwdArgs &a, cudaStream_t st, int nb = 1) { DISPATCH_N(N, launch_fwd_n, a, st, nb) }
static int launch_inv(int N, const InvArgs &a, cudaStream_t st, int nb = 1) { DISPATCH_N(N, launch_inv_n, a, st, nb) }
static int launch_level0(int N, const L0Args &a, cudaStream_t st) { DISPATCH_N(N, launch_level0_n, a, st) }

static void launch_mac(const MacArgs &a, int n_sel, bool shared_h, const char *prof_name, cudaStream_t st)
{
	if (n_sel <= 0) return;
	static const int want = getenv("DSP_B200_FIR_MAC_THREADS") ? atoi(getenv("DSP_B200_FIR_MAC_THREADS")) : 256;
	int threads = (want == 128 || want == 64) ? want : 256;
	if (a.N < threads) threads = a.N;
	dim3 grid(a.N / threads, n_sel);
	ProfScope prof(prof_name, st);
	if (shared_h) LAUNCH(k_fir_mac<true>, grid, threads, 0, st, a);
	else LAUNCH(k_fir_mac<false>, grid, threads, 0, st, a);
}

// ------------------------------------------------------------------------------------------
// unit-test hooks (tests/ only): packed real FFT round trip
// ------------------------------------------------------------------------------------------
void fir_debug_serialize(int on) { g_fir_serialize.store(on ? 1 : 0); }

int fir_debug_stall(int roles, int us, int period, int phase)
{
	const int all = DSPB200_STALL_MAIN | DSPB200_STALL_SIDE | DSPB200_STALL_SIDE2 | DSPB200_STALL_HOT;
	if (roles & ~all || us < 0 || us > FIR_STALL_MAX_US || period < 1 || period > 0xfffff || phase < 0 || phase >= period) {
		set_error("debug_stall: roles %d, %d us (at most %d), period %d, phase %d", roles, us, FIR_STALL_MAX_US, period, phase);
		return -1;
	}
	g_fir_stall.store(roles ? (unsigned long long) roles | (unsigned long long) us << 8 | (unsigned long long) period << 24 |
	                          (unsigned long long) phase << 44 : 0ULL);
	return 0;
}

int test_rfft(int B, int n_ch, const double *d_in, double *d_spec, cudaStream_t st)
{
	FwdArgs a = {};
	a.in = d_in; a.ch_stride = B; a.valid = B;
	a.spec = reinterpret_cast<double2 *>(d_spec); a.spec_ch_stride = B; a.slot = 0;
	a.tw = twiddles_2n(B);
	a.ptw = twiddles_pass(B);
	if (!a.tw || !a.ptw) return -1;
	a.n_ch = n_ch;
	return launch_fwd(B, a, st);
}

int test_irfft(int B, int n_ch, const double *d_spec, double *d_out2B, cudaStream_t st)
{
	// first half -> out[ch][0:B) (carry is zeroed scratch), second half -> out[ch][B:2B)
	double *carry = dev_alloc<double>((size_t) n_ch * B);
	if (!carry) return -1;
	InvArgs a = {};
	a.Y = reinterpret_cast<const double2 *>(d_spec);
	a.out = d_out2B; a.out_ch_stride = 2L * B;
	a.carry = carry; a.flags = INV_OUT | INV_UPDATE_CARRY;
	a.tw = twiddles_2n(B);
	a.ptw = twiddles_pass(B);
	a.n_ch = n_ch;
	int r = (a.tw && a.ptw) ? launch_inv(B, a, st) : -1;
	if (r == 0) {
		for (int c = 0; c < n_ch && r == 0; ++c)
			if (cudaMemcpyAsync(d_out2B + (size_t) c * 2 * B + B, carry + (size_t) c * B, B * sizeof(double), cudaMemcpyDeviceToDevice, st) != cudaSuccess) r = -1;
	}
	cudaStreamSynchronize(st);
	dev_free(carry);
	return r;
}

// ------------------------------------------------------------------------------------------
// operator
// ------------------------------------------------------------------------------------------
struct FirLevel {
	const double2 *tw = nullptr, *ptw = nullptr;
	double2 *fdl = nullptr, *H = nullptr;
	double *carry = nullptr, *pend = nullptr;
	long blk = 0;                 // completed blocks of this level
};

struct FirOp : Op {
	// description (host)
	std::vector<int> h_ch_map;          // selected channel -> channel index in the slab
	std::vector<double> h_taps;         // [fc][filter_frames] per-column contiguous (kept until planned)
	int fc = 1;                         // filter channels: 1 (shared) or n_sel
	long filter_frames = 0;
	long latency = 0;
	int n_sel = 0;
	bool multilevel = true;
	bool direct_io = !(getenv("DSP_B200_FIR_NO_DIRECT") && getenv("DSP_B200_FIR_NO_DIRECT")[0] == '1');

	// plan (fir_plan.h) and, per level, what it allocated
	bool planned = false;
	FirSchedule s;
	FirLevel lv[FIR_MAX_LEVELS];

	// device state
	int *d_ch_map = nullptr;
	double *d_hist = nullptr, *d_ytmp = nullptr, *d_pre = nullptr, *d_h0 = nullptr;
	double2 *d_Y = nullptr;              // [n_sel][max B]
	double2 *d_Y_side = nullptr;         // [n_sel][B last]: the tail spectrum of the next block period (side stream); two of them when level 0 has the tail
	int pipe_evict_first = getenv("DSP_B200_FIR_PIPE_EVICT") ? atoi(getenv("DSP_B200_FIR_PIPE_EVICT")) : 1;
	int pipe_fake_io = getenv("DSP_B200_FIR_PIPE_FAKEIO") ? atoi(getenv("DSP_B200_FIR_PIPE_FAKEIO")) : 0;   // measurement only
	int pipe_no_items = getenv("DSP_B200_FIR_PIPE_NOITEMS") ? atoi(getenv("DSP_B200_FIR_PIPE_NOITEMS")) : 0;   // measurement only
	long long *d_stats = nullptr;        // DSP_B200_FIR_PIPE_STATS: per-CTA cycle counters of the last pipeline launch
	bool last_block_piped = false;
	int batch_threads = getenv("DSP_B200_FIR_BATCH_THREADS") ? atoi(getenv("DSP_B200_FIR_BATCH_THREADS")) : 256;
	double *d_ring = nullptr, *d_ltmp = nullptr;
	// side stream: the upper levels' partition-0 kernels and the last level's tail MAC overlap the main stream
	cudaStream_t side = nullptr;
	cudaEvent_t ev_main = nullptr, ev_urgent = nullptr;
	// batch tiers: V spectra of the near tier and of the far tier (FirSchedule::v_slots), on a second side stream
	double2 *d_V = nullptr, *d_V2 = nullptr;
	cudaStream_t side2 = nullptr;
	// the tail's event rings and what they hold (fir_tail_steps)
	cudaEvent_t ev_tail[FIR_N_EV_TAIL] = {}, ev_batch[FIR_N_EV_BATCH] = {}, ev_bs[FIR_N_EV_BS] = {};
	FirTailRing ring;
	cudaEvent_t ev_join[2] = { nullptr, nullptr };
	cudaStream_t hot = nullptr;          // FirSchedule::hot
	cudaEvent_t ev_hot_in = nullptr, ev_hot_out = nullptr;
	bool urgent_pending = false;
	long ltmp_cap = 0;
	bool cluster_ok = false;   // selected channels are contiguous, start on an even channel, and come in fours
	double2 *d_Ybulk = nullptr;
	double *d_lo = nullptr, *d_hi = nullptr;
	long abs_pos = 0;                    // frames consumed so far (level-0 block = abs_pos / B0, offset = abs_pos % B0)
	bool pre_valid = false;
	// which paths the stream took since the last plan() (describe() "paths"): level-0 blocks completed by the fused kernel
	// (per-channel form / cluster form), the pipeline kernel, the bulk form and the general path (forward, MAC, inverse),
	// and launches of the head kernel (ragged calls)
	long n_fused = 0, n_cluster = 0, n_pipe = 0, n_bulk = 0, n_general = 0, n_head = 0;
	FirStall stall;   // dspb200_debug_stall() as it was at the start of the current level-0 block

	// the test hook's delay on stream `st` (role DSPB200_STALL_*) before its first FIR launch of level-0 block `blk`
	void stall_on(int role, long blk, cudaStream_t st)
	{
		if (!stall.hits(role, blk)) return;
		ProfScope prof("fir_stall", st);
		LAUNCH(k_fir_stall, 1, 1, 0, st, (long long) stall.us * 1000);
	}

	const char *name() const override { return "fir"; }

	std::string describe() const override
	{
		char buf[1024];
		snprintf(buf, sizeof(buf), "{\"op\":\"fir\",\"taps\":%ld,\"n_sel\":%d,\"filter_channels\":%d,\"latency\":%ld,\"planned\":%d,%s,"
		         "\"replans\":%d,\"paths\":{\"fused\":%ld,\"cluster\":%ld,\"pipe\":%ld,\"bulk\":%ld,\"general\":%ld,\"head\":%ld}}",
		         filter_frames, n_sel, fc, latency, planned ? 1 : 0, fir_schedule_json(s).c_str(), replans, n_fused, n_cluster, n_pipe, n_bulk,
		         n_general, n_head);
		return buf;
	}

	// everything plan() made: streams, events, spectra, work buffers (the description, d_ch_map and the host taps stay)
	void free_plan()
	{
		for (cudaStream_t *q : { &side, &side2, &hot })
			if (*q) { cudaStreamSynchronize(*q); cudaStreamDestroy(*q); *q = nullptr; }
		for (cudaEvent_t *e : { &ev_hot_in, &ev_hot_out, &ev_join[0], &ev_join[1], &ev_main, &ev_urgent })
			if (*e) { cudaEventDestroy(*e); *e = nullptr; }
		auto destroy = [](auto &es) { for (cudaEvent_t &e : es) { if (e) cudaEventDestroy(e); e = nullptr; } };
		destroy(ev_tail); destroy(ev_batch); destroy(ev_bs);
		ring = {};
		for (FirLevel &L : lv) { dev_free(L.fdl); dev_free(L.H); dev_free(L.carry); dev_free(L.pend); L = FirLevel(); }
		dev_free(d_V); dev_free(d_V2); dev_free(d_Y_side); dev_free(d_hist); dev_free(d_ytmp); dev_free(d_pre); dev_free(d_h0);
		dev_free(d_Y); dev_free(d_ring); dev_free(d_ltmp); dev_free(d_Ybulk); dev_free(d_lo); dev_free(d_hi); dev_free(d_stats);
		d_V = d_V2 = d_Y_side = d_Y = d_Ybulk = nullptr; d_hist = d_ytmp = d_pre = d_h0 = d_ring = d_ltmp = d_lo = d_hi = nullptr; d_stats = nullptr;
		ltmp_cap = 0; urgent_pending = false; pre_valid = false; abs_pos = 0; planned = false;
		s = FirSchedule{};
	}

	~FirOp() override
	{
		free_plan();
		dev_free(d_ch_map);
		dev_free(d_replay);
	}

	// the schedule fir_schedule() picks for calls of `hint` frames, then what it needs: spectra, rings, streams, events
	int plan(long hint, cudaStream_t st)
	{
		const FirKnobs k = FirKnobs::from_env();
		s = fir_schedule({ filter_frames, hint, n_sel, sm_count(), multilevel, direct_io }, k);
		n_fused = n_cluster = n_pipe = n_bulk = n_general = n_head = 0;
		const long T = filter_frames;
		const int nh = (fc == 1) ? 1 : n_sel;
		for (int l = 0; l < s.n_levels; ++l) {
			FirLevel &L = lv[l];
			const FirLevelPlan &Lp = s.lv[l];
			L.tw = twiddles_2n(Lp.B);
			L.ptw = twiddles_pass(Lp.B);
			if (!L.tw || !L.ptw) return -1;
			L.fdl = dev_alloc<double2>((size_t) n_sel * Lp.R * Lp.B);
			L.H = dev_alloc<double2>((size_t) nh * Lp.P * Lp.B);
			L.carry = dev_alloc<double>((size_t) n_sel * Lp.B);
			if (l > 0) L.pend = dev_alloc<double>((size_t) n_sel * Lp.B);
			if (!L.fdl || !L.H || !L.carry || (l > 0 && !L.pend)) return -1;
		}
		auto stream = [](cudaStream_t &q, int prio) { CUDA_TRY(cudaStreamCreateWithPriority(&q, cudaStreamNonBlocking, prio), return false); return true; };
		auto events = [](std::initializer_list<cudaEvent_t *> es) { for (cudaEvent_t *e : es) CUDA_TRY(cudaEventCreateWithFlags(e, cudaEventDisableTiming), return false); return true; };
		auto ring_events = [&](auto &es) { for (cudaEvent_t &e : es) if (!events({ &e })) return false; return true; };
		const size_t rows = (size_t) n_sel * s.lv[s.n_levels - 1].B;
		int lo = 0, hi = 0;
		cudaDeviceGetStreamPriorityRange(&lo, &hi);
		if (s.n_levels > 1 || s.tail_pf > 0) {
			// multi-level plans: the side stream carries the upper levels' block kernels, which must not queue behind the
			// batched MAC's CTAs; single-level plans only keep look-ahead MACs there: lowest priority.
			// (DSP_B200_FIR_MAC_PRIO: measurement -- the per-block MAC between the fused kernel and the batch tiers)
			int side_prio = (s.n_levels > 1) ? hi : lo;
			if (k.mac_prio) side_prio = (*k.mac_prio < hi) ? hi : (*k.mac_prio > lo) ? lo : *k.mac_prio;
			if (!stream(side, side_prio) || !events({ &ev_main, &ev_urgent })) return -1;
		}
		if (s.hot && (!stream(hot, hi) || !events({ &ev_hot_in, &ev_hot_out }))) return -1;
		if (s.t_batch > 0 && !(d_V = dev_alloc<double2>(s.v_slots(0) * rows))) return -1;
		if (s.t_batch > 0 && !s.use_pipe && (!stream(side2, lo) || !ring_events(ev_batch))) return -1;
		if (s.t_far > 0 && !(d_V2 = dev_alloc<double2>(s.v_slots(1) * rows))) return -1;
		if (s.t_batch > 0 && !s.use_pipe && s.tail_pf == 2 && !ring_events(ev_bs)) return -1;
		if (s.use_pipe && k.pipe_stats) d_stats = dev_alloc<long long>(8 * 1024);
		if (s.tail_pf > 0 && !s.use_pipe && !s.fold) {
			if (!(d_Y_side = dev_alloc<double2>(s.y_slots() * rows))) return -1;
			if (s.tail_pf == 2 && !ring_events(ev_tail)) return -1;
		}
		const int B0 = s.B0;
		if (s.nb_max > 1) {
			d_Ybulk = dev_alloc<double2>((size_t) s.nb_max * n_sel * B0, false);
			d_lo = dev_alloc<double>((size_t) s.nb_max * n_sel * B0, false);
			d_hi = dev_alloc<double>((size_t) s.nb_max * n_sel * B0, false);
			if (!d_Ybulk || !d_lo || !d_hi) return -1;
		}
		d_hist = dev_alloc<double>((size_t) n_sel * s.hist_len);
		d_ytmp = dev_alloc<double>((size_t) n_sel * B0);
		d_pre = dev_alloc<double>((size_t) n_sel * B0);
		d_Y = dev_alloc<double2>((size_t) n_sel * s.Bmax);
		d_h0 = dev_alloc<double>((size_t) nh * B0);
		if (latency > 0) d_ring = dev_alloc<double>((size_t) latency * n_sel);
		if (!d_hist || !d_ytmp || !d_pre || !d_Y || !d_h0 || (latency > 0 && !d_ring)) return -1;

		// filter spectra H_l[c][p] = RFFT_2B(taps[tap0 + pB : tap0 + (p+1)B) of column c), cf. fir_p.c:482-498
		double *d_taps = dev_alloc<double>((size_t) nh * T, false);
		if (!d_taps) return -1;
		CUDA_TRY(cudaMemcpyAsync(d_taps, h_taps.data(), (size_t) nh * T * sizeof(double), cudaMemcpyHostToDevice, st), return -1);
		for (int l = 0; l < s.n_levels; ++l) {
			const FirLevelPlan &Lp = s.lv[l];
			for (int p = 0; p < Lp.P; ++p) {
				FwdArgs a = {};
				const long t0 = Lp.tap0 + (long) p * Lp.B;
				a.in = d_taps + t0; a.ch_stride = T;
				a.valid = Lp.tap1 - t0;
				if (a.valid > Lp.B) a.valid = Lp.B;
				a.spec = lv[l].H; a.spec_ch_stride = (long) Lp.P * Lp.B; a.slot = p; a.tw = lv[l].tw; a.ptw = lv[l].ptw; a.n_ch = nh;
				if (launch_fwd(Lp.B, a, st)) return -1;
			}
		}
		// time-domain head taps h0[c][0:B0)
		std::vector<double> h0((size_t) nh * B0, 0.0);
		for (int c = 0; c < nh; ++c)
			for (long i = 0; i < B0 && i < T; ++i) h0[(size_t) c * B0 + i] = h_taps[(size_t) c * T + i];
		CUDA_TRY(cudaMemcpyAsync(d_h0, h0.data(), h0.size() * sizeof(double), cudaMemcpyHostToDevice, st), return -1);
		CUDA_TRY(cudaStreamSynchronize(st), return -1);
		dev_free(d_taps);
		planned = true;   // the host taps stay: a plan made from an unrepresentative first call is redone once (maybe_replan)
		return 0;
	}

	int debug_read(long long *out, int max) override
	{
		if (!d_stats || max <= 0) return 0;
		const int n = (max < 8 * 1024) ? max : 8 * 1024;
		cudaDeviceSynchronize();
		if (cudaMemcpy(out, d_stats, (size_t) n * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
		return n;
	}

	int join(cudaStream_t st) override
	{
		cudaStream_t ss[2] = { side, side2 };
		for (int i = 0; i < 2; ++i) {
			if (!ss[i]) continue;
			if (!ev_join[i]) CUDA_TRY(cudaEventCreateWithFlags(&ev_join[i], cudaEventDisableTiming), return -1);
			CUDA_TRY(cudaEventRecord(ev_join[i], ss[i]), return -1);
			CUDA_TRY(cudaStreamWaitEvent(st, ev_join[i], 0), return -1);
		}
		return 0;
	}

	void reset(cudaStream_t st) override
	{
		abs_pos = 0; pre_valid = false; urgent_pending = false;
		replay_frames = 0;
		replay_open = replans < 2;
		if (!planned) return;
		if (side) cudaStreamSynchronize(side);
		if (side2) cudaStreamSynchronize(side2);
		if (d_V) cudaMemsetAsync(d_V, 0, (size_t) s.v_slots(0) * n_sel * s.lv[s.n_levels - 1].B * sizeof(double2), st);
		if (d_V2) cudaMemsetAsync(d_V2, 0, (size_t) s.v_slots(1) * n_sel * s.lv[s.n_levels - 1].B * sizeof(double2), st);
		ring = {};
		for (int l = 0; l < s.n_levels; ++l) {
			FirLevel &L = lv[l];
			const FirLevelPlan &Lp = s.lv[l];
			L.blk = 0;
			cudaMemsetAsync(L.fdl, 0, (size_t) n_sel * Lp.R * Lp.B * sizeof(double2), st);
			cudaMemsetAsync(L.carry, 0, (size_t) n_sel * Lp.B * sizeof(double), st);
			if (L.pend) cudaMemsetAsync(L.pend, 0, (size_t) n_sel * Lp.B * sizeof(double), st);
		}
		cudaMemsetAsync(d_hist, 0, (size_t) n_sel * s.hist_len * sizeof(double), st);
		if (d_ring) cudaMemsetAsync(d_ring, 0, (size_t) latency * n_sel * sizeof(double), st);
	}

	void mac(int l, int p0, int p1, long slot_blk, cudaStream_t st, double2 *Y = nullptr, const double2 *init = nullptr)
	{
		const FirLevel &L = lv[l];
		const FirLevelPlan &Lp = s.lv[l];
		MacArgs m = {};
		m.fdl = L.fdl; m.H = L.H; m.Y = Y ? Y : d_Y; m.init = init; m.N = Lp.B; m.P = Lp.R;   // the kernel's P: rows of the ring
		m.slot0 = (int) (slot_blk % Lp.R); m.p0 = p0; m.p1 = p1;
		m.h_ch_stride = (fc == 1) ? 0 : (long) Lp.P * Lp.B;
		// the last level carries (almost) all the taps: it is the kernel the roofline line is about
		launch_mac(m, n_sel, fc == 1, (l == s.n_levels - 1) ? "fir_mac" : "fir_mac_head", st);
	}

	// block `L.blk` of level L is complete in the history ring: X into the FDL, S = MAC, IRFFT.
	// flags/out as for k_fir_inv.
	int level_block(int l, double *out, long out_ch_stride, int inv_flags, cudaStream_t st)
	{
		FirLevel &L = lv[l];
		const FirLevelPlan &Lp = s.lv[l];
		FwdArgs f = {};
		f.in = d_hist + (L.blk * Lp.B) % s.hist_len; f.ch_stride = s.hist_len; f.valid = Lp.B;
		f.spec = L.fdl; f.spec_ch_stride = (long) Lp.R * Lp.B; f.slot = (int) (L.blk % Lp.R); f.tw = L.tw; f.ptw = L.ptw; f.n_ch = n_sel;
		if (launch_fwd(Lp.B, f, st)) return -1;
		mac(l, 0, Lp.P, L.blk, st);
		InvArgs v = {};
		v.Y = d_Y; v.out = out; v.out_ch_stride = out_ch_stride; v.carry = L.carry; v.flags = inv_flags; v.tw = L.tw; v.ptw = L.ptw; v.n_ch = n_sel;
		if (launch_inv(Lp.B, v, st)) return -1;
		++L.blk;
		return 0;
	}

	// After level 0 finished a block: every larger level whose block just completed is advanced -- on the
	// SIDE stream, so that the caller's stream (and, in host mode, the D2H of the block just produced and
	// the H2D of the next one) is not held up:
	//   - the level's result for the block period that starts now is due at once: fused kernel (spectrum
	//     into the level's FDL, S = X_q H_0 + Y_q, inverse, result into `pend`), `ev_urgent` tells the main
	//     stream when it is there;
	//   - Y_q = sum_{p>=1} X_{q-p} H_p (last level only) involves blocks that were complete one period
	//     earlier: Y_{q+1} is launched right now and consumed by the fused kernel of the NEXT period, so the
	//     HBM-streaming MAC has a whole period to overlap with the FFT kernels.
	int advance_upper_levels(cudaStream_t st)
	{
		// Everything goes to the side stream: in host mode the D2H of this block and the H2D of the next are not
		// held up, and in device-resident mode it is faster too than with the partition-0 kernels on the caller's
		// stream: the caller's stream keeps only stash, level 0, unstash.
		const bool serial = g_fir_serialize.load(std::memory_order_relaxed) != 0;
		cudaStream_t us = serial ? st : side;
		bool any = false;
		for (int l = 1; l < s.n_levels; ++l) {
			FirLevel &L = lv[l];
			const FirLevelPlan &Lp = s.lv[l];
			if (abs_pos % Lp.B != 0) break;   // sizes double: if this one is not complete, none above is
			if (!any && us != st) {
				CUDA_TRY(cudaEventRecord(ev_main, st), return -1);
				CUDA_TRY(cudaStreamWaitEvent(side, ev_main, 0), return -1);
				stall_on(DSPB200_STALL_SIDE, lv[0].blk - 1, side);
			}
			any = true;
			L0Args f = {};
			f.in = d_hist + (L.blk * Lp.B) % s.hist_len; f.in_ch_stride = s.hist_len;
			f.fdl = L.fdl; f.fdl_ch_stride = (long) Lp.R * Lp.B; f.fdl_rows = Lp.R;
			f.H = L.H; f.h_ch_stride = (fc == 1) ? 0 : (long) Lp.P * Lp.B;
			f.P = 1; f.slot = (int) (L.blk % Lp.R);
			f.out = L.pend; f.out_ch_stride = Lp.B; f.carry = L.carry; f.tw = L.tw; f.ptw = L.ptw; f.n_ch = n_sel;
			f.init = (Lp.tail && L.blk >= 1) ? d_Y_side : nullptr;   // Y of this block: launched one period ago, same stream
			if (launch_level0(Lp.B, f, us)) return -1;
			++L.blk;
		}
		if (!any) return 0;
		CUDA_TRY(cudaEventRecord(ev_urgent, us), return -1);
		urgent_pending = (us != st);
		if (abs_pos % s.Bmax != 0) return 0;   // the last level's block is not complete
		return launch_tail(lv[s.n_levels - 1].blk - 1, st, us, serial ? st : side2);
	}

	// the event of a FirEv (FirEvRing order), and slot i of a ring of spectra of the tail level (FirSchedule::v_slots)
	cudaEvent_t event(const FirEv &e) const
	{
		const cudaEvent_t *rings[] = { nullptr, &ev_main, &ev_urgent, ev_tail, ev_batch, ev_bs };
		return rings[e.ring][e.slot];
	}
	double2 *slot(double2 *spectra, int i) const { return spectra + (size_t) i * n_sel * s.lv[s.n_levels - 1].B; }
	int wait(cudaStream_t st, const FirEv &e)
	{
		if (e.ring != FIR_EV_NONE) CUDA_TRY(cudaStreamWaitEvent(st, event(e), 0), return -1);
		return 0;
	}

	// The launches after block q of the tail level (fir_tail_steps), the side roles on ts and bs; either may be the caller's
	// stream st, which then has no ev_main to wait for.  The stall hook delays a side stream where it starts on the block.
	int launch_tail(long q, cudaStream_t st, cudaStream_t ts, cudaStream_t bs)
	{
		const FirLevel &L = lv[s.n_levels - 1];
		const FirLevelPlan &Lp = s.lv[s.n_levels - 1];
		const FirTailSteps steps = fir_tail_steps(s, q, n_sel, ring);
		for (int i = 0; i < steps.n; ++i) {
			const FirTailStep &x = steps.l[i];
			cudaStream_t xs = (x.role == FIR_SIDE2) ? bs : ts;
			for (const FirEv &w : x.wait)
				if (!(w.ring == FIR_EV_MAIN && xs == st) && wait(xs, w)) return -1;
			if ((x.wait[0].ring == FIR_EV_MAIN || x.wait[0].ring == FIR_EV_URGENT) && xs != st)
				stall_on((x.role == FIR_SIDE2) ? DSPB200_STALL_SIDE2 : DSPB200_STALL_SIDE, lv[0].blk - 1, xs);
			double2 *Y = (x.kind != FIR_TAIL_TIER) ? slot(d_Y_side, x.y) : nullptr;
			const double2 *V = (x.v >= 0) ? slot(d_V, x.v) : nullptr;
			if (x.kind == FIR_TAIL_MAC) mac(s.n_levels - 1, s.mac_parts().first, s.mac_parts().second, x.j, xs, Y, V);
			else if (x.kind == FIR_TAIL_TIER) {
				int threads = batch_threads_for(x.d.T);
				if (s.n_levels == 1 && (batch_threads == 128 || batch_threads == 64) && batch_threads < threads) threads = batch_threads;
				if (Lp.B < threads) threads = Lp.B;
				// whole launches of the far tier: at most one CTA per SM (DSP_B200_FIR_FAR_SMEM_KB, 0 = no cap)
				static const long far_kb = getenv("DSP_B200_FIR_FAR_SMEM_KB") ? atol(getenv("DSP_B200_FIR_FAR_SMEM_KB")) : 0;
				launch_mac_batch(x.d.T, fc == 1, dim3(Lp.B / threads, x.d.rows + x.d.pass_rows), threads, xs, batch_args(x.d, q),
				                 x.d.tier ? "fir_mac_batch_far" : "fir_mac_batch", (x.d.tier && !s.stagger && far_kb > 0) ? (size_t) far_kb * 1024 : 0);
			}
			else {
				// one grid for the per-block MAC and this block's class of the near tier
				TailArgs ta = {};
				ta.m.fdl = L.fdl; ta.m.H = L.H; ta.m.Y = Y; ta.m.init = V;
				ta.m.N = Lp.B; ta.m.P = Lp.R; ta.m.slot0 = (int) (x.j % Lp.R); ta.m.p0 = s.mac_parts().first; ta.m.p1 = s.mac_parts().second;
				ta.m.h_ch_stride = (fc == 1) ? 0 : (long) Lp.P * Lp.B;
				ta.b = batch_args(x.d, q);
				ta.n_batch_y = x.d.rows;
				const dim3 grid(Lp.B / 256, ta.n_batch_y + n_sel);
				ProfScope prof("fir_tail", xs);
				if (fc == 1) LAUNCH((k_fir_tail<4, true>), grid, 256, 0, xs, ta);
				else LAUNCH((k_fir_tail<4, false>), grid, 256, 0, xs, ta);
			}
			for (const FirEv &e : x.rec)
				if (e.ring != FIR_EV_NONE) CUDA_TRY(cudaEventRecord(event(e), xs), return -1);
		}
		return 0;
	}

	// the arguments of a tier launch after block q of the tail level
	MacBatchArgs batch_args(const FirTierLaunch &d, long q) const
	{
		const FirLevel &L = lv[s.n_levels - 1];
		const FirLevelPlan &Lp = s.lv[s.n_levels - 1];
		MacBatchArgs b = {};
		b.fdl = L.fdl; b.H = L.H; b.N = Lp.B; b.P = Lp.P; b.n_sel = n_sel; b.q = q;
		b.V = d.tier ? d_V2 : d_V; b.n_slots = s.v_slots(d.tier);
		b.h_ch_stride = (fc == 1) ? 0 : (long) Lp.P * Lp.B;
		b.pf = d.pf; b.p_lo = d.p_lo; b.p_hi = d.p_hi; b.g = d.g; b.K = d.K; b.w = d.w;
		if (d.from_far) { b.Vin = d_V2; b.vin_slots = s.v_slots(1); }
		if (d.pass_rows > 0) { b.n_tier_y = d.rows; b.pass_g = d.pass_g; b.pass_m = d.pass_m; }
		return b;
	}

	// Single-level plans: after block q of level 0 has entered the FDL (fused kernel or general path), the part
	// of block q+2's spectrum that is already known, Y_{q+2} = sum_{p>=2} X_{q+2-p} H_p, is accumulated on the
	// side stream -- a whole block period ahead of the fused kernel that adds X_{q+2} H_0 + X_{q+1} H_1 to it.
	// With time-batching, V_j = sum_{p>=T+2} (T periods per launch, second side stream) is its starting value.
	int advance_tail0(cudaStream_t st)
	{
		const FirLevel &L = lv[0];
		const FirLevelPlan &Lp = s.lv[0];
		const bool serial = g_fir_serialize.load(std::memory_order_relaxed) != 0;
		// The per-block MAC runs on the side stream, time-slicing with the next fused kernel (a shorter step than with
		// the MAC queued behind the fused kernel on the caller's stream, where it runs alone -- DSP_B200_FIR_TAIL_MAIN=1
		// selects that for measurements).
		static const int tail_main = getenv("DSP_B200_FIR_TAIL_MAIN") ? atoi(getenv("DSP_B200_FIR_TAIL_MAIN")) : -1;
		const long q = L.blk - 1;
		if (s.use_pipe) {
			// The pipeline kernel of block q does block q's share of the batched tail itself (channels of residue
			// q % 4: V_{q+2} .. V_{q+5} from the blocks up to q-1).  A block that took the general path gets the same
			// share from the stand-alone batch kernel, here, on the caller's stream.
			if (s.t_batch > 0 && !last_block_piped && q >= 1) {
				const int T = s.t_batch, g = (int) (q % T), rows = fir_class_rows(n_sel, g, T, 1);
				if (rows > 0) {
					const int threads = (Lp.B < batch_threads_for(T)) ? Lp.B : batch_threads_for(T);
					const FirTierLaunch d = { 0, T, g, T, 1, 2, T + 2, Lp.P, rows, false, 0, 0, 0 };
					launch_mac_batch(T, fc == 1, dim3(Lp.B / threads, rows), threads, st, batch_args(d, q - 1));
				}
			}
			return 0;
		}
		if (!serial) CUDA_TRY(cudaEventRecord(ev_main, st), return -1);
		return launch_tail(q, st, (serial || tail_main > 0) ? st : side, serial ? st : side2);
	}

	// What the unstash / head kernels add on top of level 0 for the frames starting at `first_frame_abs`:
	// every upper level's result for its current block period.
	PendArgs pend_args(long first_frame_abs) const
	{
		PendArgs p = {};
		for (int l = 1; l < s.n_levels; ++l) {
			const FirLevel &L = lv[l];
			p.buf[p.n] = L.pend; p.len[p.n] = s.lv[l].B; p.off[p.n] = (int) (first_frame_abs % s.lv[l].B);
			++p.n;
		}
		return p;
	}

	// the main stream waits for the upper levels' kernels right before the first kernel that reads `pend`
	void side_wait(long, cudaStream_t st)
	{
		if (urgent_pending) {
			cudaStreamWaitEvent(st, ev_urgent, 0);
			urgent_pending = false;
		}
	}

	// nb whole level-0 blocks of one call (single-level plans): stash all, ONE forward launch, ONE pass over
	// the FDL and the filter spectra for all nb outputs (k_fir_mac_bulk), ONE inverse launch, ONE overlap/scatter
	int bulk_blocks(int nb, const double *src, double *d, long dstride, const int *dmap, cudaStream_t st)
	{
		FirLevel &L = lv[0];
		const FirLevelPlan &Lp = s.lv[0];
		const long C = channels;
		const long off = (abs_pos % s.hist_len);
		// the new frames join the history ring (it holds nb_max blocks; at most one wrap)
		{
			const long total = (long) nb * s.B0, first = (total < s.hist_len - off) ? total : s.hist_len - off;
			dim3 grid(ceil_div(first, 32), ceil_div(n_sel, 32));
			LAUNCH(k_fir_stash, grid, 256, 0, st, src, C, d_ch_map, d_hist, s.hist_len, off, (int) first, n_sel);
			if (first < total) {
				dim3 grid2(ceil_div(total - first, 32), ceil_div(n_sel, 32));
				LAUNCH(k_fir_stash, grid2, 256, 0, st, src + first * C, C, d_ch_map, d_hist, s.hist_len, 0L, (int) (total - first), n_sel);
			}
		}
		FwdArgs f = {};
		f.in = d_hist; f.ch_stride = s.hist_len; f.valid = s.B0;
		f.spec = L.fdl; f.spec_ch_stride = (long) Lp.R * s.B0; f.slot = (int) (L.blk % Lp.R); f.tw = L.tw; f.ptw = L.ptw; f.n_ch = n_sel;
		f.ring_len = s.hist_len; f.ring_off = off; f.slot_rows = Lp.R;
		if (launch_fwd(s.B0, f, st, nb)) return -1;
		{
			MacBulkArgs b = {};
			b.fdl = L.fdl; b.H = L.H; b.Y = d_Ybulk; b.N = s.B0; b.P = Lp.P; b.rows = Lp.R; b.n_sel = n_sel; b.nb = nb; b.j = L.blk;
			b.h_ch_stride = (fc == 1) ? 0 : (long) Lp.P * s.B0;
			const int threads = (s.B0 < 256) ? s.B0 : 256;
			dim3 grid(s.B0 / threads, n_sel);
			ProfScope prof("fir_mac_bulk", st);
			if (fc == 1) LAUNCH((k_fir_mac_bulk<FIR_NB_MAX, true>), grid, threads, 0, st, b);
			else LAUNCH((k_fir_mac_bulk<FIR_NB_MAX, false>), grid, threads, 0, st, b);
		}
		InvArgs v = {};
		v.Y = d_Ybulk; v.out = d_lo; v.out_ch_stride = s.B0; v.carry = d_hi; v.flags = INV_RAW; v.tw = L.tw; v.ptw = L.ptw; v.n_ch = n_sel;
		if (launch_inv(s.B0, v, st, nb)) return -1;
		{
			dim3 grid(ceil_div(s.B0, 32), ceil_div(n_sel, 32), nb);
			LAUNCH(k_fir_unstash_bulk, grid, 256, 0, st, d_lo, d_hi, L.carry, s.B0, d, dstride, dmap, n_sel);
		}
		CUDA_TRY(cudaMemcpyAsync(L.carry, d_hi + (size_t) (nb - 1) * n_sel * s.B0, (size_t) n_sel * s.B0 * sizeof(double), cudaMemcpyDeviceToDevice, st), return -1);
		L.blk += nb;
		n_bulk += nb;
		pre_valid = false;
		return 0;
	}

	int ensure_pre(cudaStream_t st)
	{
		if (pre_valid) return 0;
		FirLevel &L = lv[0];
		mac(0, 1, s.lv[0].P, L.blk, st);   // R: completed level-0 blocks only
		InvArgs v = {};
		v.Y = d_Y; v.out = d_pre; v.out_ch_stride = s.B0; v.carry = L.carry; v.flags = INV_OUT; v.tw = L.tw; v.ptw = L.ptw; v.n_ch = n_sel;
		if (launch_inv(s.B0, v, st)) return -1;
		pre_valid = true;
		return 0;
	}

	// ---- re-planning ---------------------------------------------------------------------------------
	// The partition size comes from the first call's frame count (or the caller's hint).  Frontends do not always
	// open with a representative call (a LADSPA host probing with a few frames, a short first read): while the stream
	// is younger than REPLAY_MAX frames its input is kept, and when a later call is at least twice the planned block
	// the plan is redone for that size and the kept input replayed through it (outputs discarded) -- the state is then
	// exactly what it would have been with the right plan from the start.
	static constexpr long REPLAY_MAX = 16384;
	double *d_replay = nullptr;      // [replay_frames][channels], interleaved as it came
	long replay_frames = 0;
	bool replay_open = true;
	int replans = 0;

	int keep_for_replay(long frames, const double *in, cudaStream_t st)
	{
		if (!replay_open) return 0;
		if (replay_frames + frames > REPLAY_MAX || replans >= 2 || s.B0 >= 4096) {
			replay_open = false;
			dev_free(d_replay);
			d_replay = nullptr;
			return 0;
		}
		if (!d_replay) {
			d_replay = dev_alloc<double>((size_t) REPLAY_MAX * channels, false);
			if (!d_replay) { replay_open = false; return 0; }   // no memory to spare: keep the first plan
		}
		CUDA_TRY(cudaMemcpyAsync(d_replay + replay_frames * channels, in, (size_t) frames * channels * sizeof(double), cudaMemcpyDeviceToDevice, st), return -1);
		replay_frames += frames;
		return 0;
	}

	int maybe_replan(long frames, cudaStream_t st)
	{
		if (!replay_open || !planned || frames < 2L * s.B0 || replay_frames == 0 && abs_pos > 0) return 0;
		if (getenv("DSP_B200_FIR_NO_REPLAN")) return 0;
		const long kept = replay_frames;
		CUDA_TRY(cudaStreamSynchronize(st), return -1);
		free_plan();
		++replans;
		if (plan(frames, st)) return -1;
		if (kept > 0) {
			double *scratch = dev_alloc<double>((size_t) kept * channels, false);
			if (!scratch) return -1;
			const bool was_open = replay_open;
			replay_open = false;   // the replay itself is not recorded again
			const long r = run_planned(kept, d_replay, scratch, st);
			replay_open = was_open;
			CUDA_TRY(cudaStreamSynchronize(st), return -1);
			dev_free(scratch);
			if (r < 0) return -1;
		}
		return 0;
	}

	long run(long frames, const double *in, double *out, cudaStream_t st) override
	{
		if (frames <= 0) return 0;
		const long C = channels;
		if (in != out && n_sel < C)
			CUDA_TRY(cudaMemcpyAsync(out, in, (size_t) frames * C * sizeof(double), cudaMemcpyDeviceToDevice, st), return -1);
		if (n_sel == 0) return frames;   // a slab the selector leaves empty: pass-through, nothing to plan (no taps were kept for it)
		if (!planned && plan(frames, st)) return -1;
		if (maybe_replan(frames, st)) return -1;
		if (keep_for_replay(frames, in, st)) return -1;
		return run_planned(frames, in, out, st);
	}

	long run_planned(long frames, const double *in, double *out, cudaStream_t st)
	{
		const long C = channels;

		// where the convolution result goes: straight to `out`, or to a compact temp when a latency ring follows
		double *dst = out;
		long dstride = C;
		const int *dmap = d_ch_map;
		if (latency > 0) {
			if (ltmp_cap < frames) {
				dev_free(d_ltmp);
				d_ltmp = dev_alloc<double>((size_t) frames * n_sel, false);
				if (!d_ltmp) return -1;
				ltmp_cap = frames;
			}
			dst = d_ltmp; dstride = n_sel; dmap = nullptr;
		}
		const long abs0 = abs_pos;
		FirLevel &L0 = lv[0];
		const FirLevelPlan &Lp0 = s.lv[0];
		const dim3 tgrid_full(ceil_div(s.B0, 32), ceil_div(n_sel, 32));

		long done = 0;
		while (done < frames) {
			const double *src = in + done * C;
			double *d = dst + done * dstride;
			if (abs_pos % s.B0 == 0) {
				stall = FirStall::load();
				stall_on(DSPB200_STALL_MAIN, L0.blk, st);
			}
			if (s.nb_max > 1 && abs_pos % s.B0 == 0 && frames - done >= 2L * s.B0) {
				long nb = (frames - done) / s.B0;
				if (nb > s.nb_max) nb = s.nb_max;
				if (bulk_blocks((int) nb, src, d, dstride, dmap, st)) return -1;
				abs_pos += nb * s.B0;
				done += nb * s.B0;
				continue;
			}
			const int pos = (int) (abs_pos % s.B0);
			const long blk_off = (abs_pos - pos) % s.hist_len;
			const int seg = (int) ((frames - done < s.B0 - pos) ? frames - done : s.B0 - pos);
			const PendArgs pend = pend_args(abs_pos);
			// single-level plans: the fused kernel reads the caller's block and writes the caller's result itself
			const bool direct = direct_io && s.n_levels == 1 && pos == 0 && seg == s.B0 && (Lp0.P <= 2 || s.tail_pf == 2);
			// the new frames join the history ring
			if (!direct) {
				dim3 grid(ceil_div(seg, 32), ceil_div(n_sel, 32));
				LAUNCH(k_fir_stash, grid, 256, 0, st, src, C, d_ch_map, d_hist, s.hist_len, blk_off + pos, seg, n_sel);
			}
			if (pos == 0 && seg == s.B0) {
				// fast path: one whole aligned block
				last_block_piped = false;
				if (s.use_pipe && direct) {
					PipeArgs f = {};
					f.xin = src; f.xin_stride = C; f.xin_map = d_ch_map;
					f.yout = d; f.yout_stride = dstride; f.yout_map = dmap;
					f.fdl = L0.fdl; f.fdl_ch_stride = (long) Lp0.R * s.B0; f.fdl_rows = Lp0.R; f.slot = (int) (L0.blk % Lp0.R);
					f.H = L0.H; f.h_ch_stride = (fc == 1) ? 0 : (long) Lp0.P * s.B0;
					f.P = Lp0.P; f.pf = s.pipe_pf;
					f.V = (s.t_batch > 0) ? d_V : nullptr; f.v_slots = s.v_slots(0); f.blk = L0.blk;
					f.carry = L0.carry; f.tw = L0.tw; f.ptw = L0.ptw; f.n_ch = n_sel;
					f.evict_first = pipe_evict_first;
					f.fake_io = (pipe_fake_io && C == n_sel && dstride == C) ? 1 : 0;
					f.no_batch_items = pipe_no_items;
					f.stats = d_stats;
					if (launch_pipe(s.B0, f, st)) return -1;
					++L0.blk;
					++n_pipe;
					last_block_piped = true;
				}
				else if (s.use_pipe) {
					// a whole block that cannot use the direct form (never happens today: direct_io is a plan-time switch)
					if (level_block(0, d_ytmp, s.B0, INV_OUT | INV_UPDATE_CARRY, st)) return -1;
					++n_general;
				}
				else if (Lp0.P <= 2 || s.tail_pf == 2) {
					L0Args f = {};
					f.in = d_hist + blk_off; f.in_ch_stride = s.hist_len;
					if (direct) {
						f.xin = src; f.xin_stride = C; f.xin_map = d_ch_map;
						f.yout = d; f.yout_stride = dstride; f.yout_map = dmap;
						// four adjacent channels per cluster: needs the selected channels contiguous and 16-byte aligned rows
						f.cluster_io = cluster_ok && s.B0 >= 2048 && C % 2 == 0 && dstride % 2 == 0 &&
						               ((reinterpret_cast<size_t>(src) | reinterpret_cast<size_t>(d)) & 15) == 0;
					}
					f.fdl = L0.fdl; f.fdl_ch_stride = (long) Lp0.R * s.B0; f.fdl_rows = Lp0.R;
					f.H = L0.H; f.h_ch_stride = (fc == 1) ? 0 : (long) Lp0.P * s.B0;
					f.P = s.l0_parts(); f.slot = (int) (L0.blk % Lp0.R);
					f.out = d_ytmp; f.out_ch_stride = s.B0; f.carry = L0.carry; f.tw = L0.tw; f.ptw = L0.ptw; f.n_ch = n_sel;
					cudaStream_t ls = st;
					// (not in a synchronous host call: it works on one block at a time, the two event hops cost it time per
					// block and the priority buys it nothing; with blocks in flight -- submit/wait -- it pays)
					const bool use_hot = hot && direct && s.tail_pf == 2 && !host_mode && !g_fir_serialize.load(std::memory_order_relaxed);
					if (use_hot) {
						CUDA_TRY(cudaEventRecord(ev_hot_in, st), return -1);
						CUDA_TRY(cudaStreamWaitEvent(hot, ev_hot_in, 0), return -1);
						ls = hot;
					}
					const FirTailRead c = fir_fused_read(s, L0.blk, ring);
					if (wait(ls, c.wait)) return -1;
					if (c.v >= 0) f.init = slot(d_V, c.v);
					if (c.y >= 0) f.init = slot(d_Y_side, c.y);
					if (s.fold) {
						f.blk = L0.blk;
						f.cls_T = s.t_batch; f.cls_K = s.stagger ? s.t_batch : 1; f.cls_w = s.class_w; f.la = s.la; f.pass_m = s.pass_m;
					}
					if (use_hot) stall_on(DSPB200_STALL_HOT, L0.blk, hot);
					if (launch_level0(s.B0, f, ls)) return -1;
					if (use_hot) {
						CUDA_TRY(cudaEventRecord(ev_hot_out, hot), return -1);
						CUDA_TRY(cudaStreamWaitEvent(st, ev_hot_out, 0), return -1);
					}
					++L0.blk;
					if (f.cluster_io) ++n_cluster;
					else ++n_fused;
				}
				else {
					if (level_block(0, d_ytmp, s.B0, INV_OUT | INV_UPDATE_CARRY, st)) return -1;
					++n_general;
				}
				if (!direct) {
					side_wait(abs_pos, st);
					LAUNCH(k_fir_unstash, tgrid_full, 256, 0, st, d_ytmp, (long) s.B0, pend, d, dstride, dmap, s.B0, n_sel);
				}
				pre_valid = false;
			}
			else {
				if (ensure_pre(st)) return -1;
				dim3 grid(ceil_div(seg, 128), n_sel);
				side_wait(abs_pos, st);
				LAUNCH(k_fir_head, grid, 128, 0, st, d_hist, s.hist_len, blk_off, d_pre, d_h0, (fc == 1) ? 0L : (long) s.B0, pend,
				       d, dstride, dmap, s.B0, pos, seg);
				++n_head;
				if (pos + seg == s.B0) {
					// block complete: X into the FDL, carry = IRFFT(S)[B:2B) (its first half has been emitted already)
					last_block_piped = false;
					if (!g_fir_serialize.load(std::memory_order_relaxed) && wait(st, fir_general_wait(L0.blk, ring))) return -1;
					if (level_block(0, nullptr, 0, INV_UPDATE_CARRY, st)) return -1;
					++n_general;
					pre_valid = false;
				}
			}
			abs_pos += seg;
			done += seg;
			if (abs_pos % s.B0 == 0 && ((s.tail_pf == 2) ? advance_tail0(st) : advance_upper_levels(st))) return -1;
		}

		if (latency > 0) {
			const long total = frames * n_sel;
			LAUNCH(k_delay_read, ceil_div(total, 256), 256, 0, st, d_ltmp, (long) n_sel, d_ring, out, C, d_ch_map, n_sel, frames, latency, abs0);
			const long cnt = (frames > latency) ? latency : frames;
			LAUNCH(k_delay_write, ceil_div(cnt * n_sel, 256), 256, 0, st, d_ltmp, (long) n_sel, d_ring, n_sel, frames, latency, abs0);
		}
		return frames;
	}
};

Op *make_fir_op(int slab_channels, int fs, const char *slab_selector, const double *taps, int filter_channels,
                long filter_frames, const int *taps_cols, long latency, long block_hint, cudaStream_t st)
{
	std::unique_ptr<FirOp> op(new FirOp());
	op->channels = slab_channels;
	op->fs_in = op->fs_out = fs;
	for (int c = 0; c < slab_channels; ++c)
		if (!slab_selector || slab_selector[c]) op->h_ch_map.push_back(c);
	op->n_sel = (int) op->h_ch_map.size();
	op->fc = (filter_channels == 1) ? 1 : op->n_sel;
	op->filter_frames = filter_frames;
	op->latency = latency;
	const char *ml = getenv("DSP_B200_FIR_LEVELS");
	op->multilevel = !(ml && ml[0] == '1' && ml[1] == '\0');
	if (op->n_sel > 0) {
		// gather this slab's columns of the filter, one contiguous row per column:
		// taps_cols[k] = column of the k-th selected channel
		op->h_taps.resize((size_t) filter_frames * op->fc);
		for (int k = 0; k < op->fc; ++k) {
			const int col = (filter_channels == 1) ? 0 : taps_cols[k];
			for (long i = 0; i < filter_frames; ++i)
				op->h_taps[(size_t) k * filter_frames + i] = taps[(size_t) i * filter_channels + col];
		}
		{
			bool contiguous = (op->n_sel % 4 == 0) && (op->h_ch_map[0] % 2 == 0);
			for (int k = 1; k < op->n_sel && contiguous; ++k) contiguous = op->h_ch_map[k] == op->h_ch_map[0] + k;
			op->cluster_ok = contiguous && !(getenv("DSP_B200_FIR_NO_CLUSTER") && getenv("DSP_B200_FIR_NO_CLUSTER")[0] == '1');
		}
		op->d_ch_map = dev_alloc<int>(op->n_sel, false);
		if (!op->d_ch_map) return nullptr;
		CUDA_TRY(cudaMemcpy(op->d_ch_map, op->h_ch_map.data(), op->n_sel * sizeof(int), cudaMemcpyHostToDevice), return nullptr);
		if (block_hint > 0 && op->plan(block_hint, st)) return nullptr;
	}
	return op.release();
}

}  // namespace dspb200
