// resample.cu -- K3: rational resampler as a polyphase FIR.
//
// Reference behaviour reproduced (/root/reference/resample.c): parameters :274-316, Albrecht
// 9-term window :52-80, norm_sinc :82-87, windowed sinc :361-364 and its spectrum :366, the
// per-block spectral image/fold multiply + overlap-add :89-152, output pacing :93-108,144-147,
// reset :154-161, drain2 :163-188.
//
// The reference works in the frequency domain on blocks of in_len frames.  Because each block
// is zero-padded to 2*in_len and the filter is shorter than in_len, that algorithm is exactly
// the linear periodically-time-varying FIR (SURVEY.md A.4, checked against the compiled
// reference to 3e-15 for 160/147, 147/160, 2/1, 1/2, 320/441 before this file was written)
//     y[m] = sum_{t=0}^{in_len-1} G[(m d) mod n][t] * x[floor(m d / n) - t]
//     G[ph][t] = g(ph + t n),
//     g(tau) = 1/(2 in_len) [ S_0 + 2 sum_{k=1}^{K-1} Re(S_k e^{i th k tau}) + Re(S_K e^{i th K tau}) ],
//     th = 2 pi / (2 in_len n),  K = sinc_len,  S = DFT_{2K}(windowed sinc)
// and the emitted stream is y[out_delay + q].  The n x in_len tap table G (0.75 MB for
// 44100->48000) is built on the device at init from the reference's own sinc samples; the hot
// kernel is a per-channel dot product with lanes along channels, so every load of the
// interleaved input is a coalesced row and the taps are broadcast loads from shared memory.
// The reference's per-call frame pacing is replayed by an integer state machine on the host
// (RsPacing, resample_plan.h), so each call emits exactly the frame count resample_effect_run() would.
#include "common.cuh"
#include "ops.h"
#include "resample_plan.h"
#include <cmath>

namespace dspb200 {

// resample_params() (resample_plan.h) with the library's message on failure
int resample_params_or_error(int fs_in, int fs_out, double bw, ResampleParams *p)
{
	const int e = resample_params(fs_in, fs_out, bw, p);
	if (e == RS_BAD_RATES) set_error("resample: bad rates %d -> %d", fs_in, fs_out);
	else if (e == RS_BAD_BANDWIDTH) set_error("resample: bandwidth out of range");
	return e ? -1 : 0;
}

// resample.c:52-80 (WINDOW_FUNCTION 3)
static double albrecht9(double x)
{
	static const double a[9] = {
		2.318028013590306028393e-1, 3.932575471789488615081e-1, 2.385434764970747429454e-1,
		1.014370437785239811268e-1, 2.911516061918003918645e-2, 5.280988177252078698806e-3,
		5.382909093381945363528e-4, 2.442086527507867730168e-5, 2.706153764205043532817e-7,
	};
	if (x >= 1.0 || x <= 0.0) return 0.0;
	double w = a[0];
	for (int i = 1; i < 9; ++i) {
		const double c = (i & 1) ? -a[i] : a[i];
		w += c * cos(2 * i * M_PI * x);
	}
	return w;
}

// S[k] = sum_i sinc[i] exp(-2 pi i i k / (2K)), k = 0..K   (what fftw r2c gives at resample.c:366)
__global__ void k_rs_sinc_dft(const double *sinc, int m_os, int K, double2 *S)
{
	const int k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k > K) return;
	double re = 0.0, im = 0.0;
	for (int i = 1; i < m_os; ++i) {
		const long r = ((long) i * k) % (2L * K);
		double sn, cs;
		sincospi((double) r / K, &sn, &cs);
		const double v = sinc[i];
		re = fma(v, cs, re);
		im = fma(-v, sn, im);
	}
	S[k] = make_double2(re, im);
}

// G[ph][t] = g(ph + t n)
__global__ void k_rs_table(const double2 *S, int K, int n, int in_len, double *G, int g_stride, int pad)
{
	const long idx = (long) blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= (long) n * in_len) return;
	const int ph = (int) (idx / in_len), t = (int) (idx % in_len);
	const long tau = ph + (long) t * n;
	const long Pd = 2L * in_len * n;
	double acc = 0.0;
	for (int k = 1; k <= K; ++k) {
		const long r = ((long) k * tau) % Pd;
		double sn, cs;
		sincospi(2.0 * (double) r / (double) Pd, &sn, &cs);
		const double2 s = S[k];
		const double term = s.x * cs - s.y * sn;
		acc += (k == K) ? 0.5 * term : term;
	}
	G[(long) ph * g_stride + pad + t] = (S[0].x + 2.0 * acc) / (2.0 * in_len);   // rows are zero-padded by `pad` on both sides
}

// out[q][c] = sum_t G[(m d) % n][t] * x[(m d) / n - t][c],  m = m0 + q;  x lives in a ring of rows.
// A CTA produces Q = R*WARPS consecutive output frames for 32*CH channels: warp w owns frames R w .. R w + R-1,
// lane = CH adjacent channels, R x CH accumulators in registers.  The Q tap windows are first gathered into
// shared memory as S[k][r] = G[ph_r][ih_r - (i_top - k)] -- row k holds the taps the Q outputs apply to
// input row i_top - k (zero where a window has not begun or has ended: the rows of G are zero-padded by
// `pad` on both sides, and S is zero past the end of the span, so the loop needs no bounds) -- in chunks of
// ROWS rows.  The warps then walk the input rows downwards once, one software-pipeline stage (RS_G rows)
// ahead of the arithmetic: every row is loaded once per warp (CH doubles per lane, coalesced; the warps of
// the CTA read the same rows within a few iterations of each other, so all but one of the loads hit in L1)
// and meets its R taps as R/2 broadcast 128-bit shared loads.
// The kernel is bound by the L1/LSU data pipe before it is bound by FP64 issue (a broadcast LDS.128 costs 2
// wavefronts, a coalesced LDG.128 about 10), so the register tile is as large as the register file allows: 16 outputs x 4
// channels = 64 accumulators per lane, 2 LDG.128 + 8 LDS.128 per 64 DFMA.
// History: (1) taps by warp-uniform global loads: the 160 phases' rows -- 0.75 MB for 44100->48000 -- do not
// fit in L1, the kernel sat on L2 latency; (2) taps in shared memory, 8 x 4 tile: LSU-bound as above.
constexpr int RS_G = 4;          // input rows per software-pipeline stage
constexpr int RS_QMAX = 64;      // most output frames per CTA of any variant (sizes the zero padding of G's rows)

template <int R, int CH, int WARPS>
struct RsCfg {
	static constexpr int Q = R * WARPS;             // output frames per CTA
	static constexpr int LD = Q + 2;                // row stride of S in doubles: 16-byte aligned rows, column stores spread over banks
	static constexpr int ROWS = (4096 / Q) & ~(RS_G - 1);   // input rows per chunk (about 32 KB of taps)
	static constexpr int THREADS = 32 * WARPS;
	static_assert(Q <= RS_QMAX && ROWS % RS_G == 0 && ROWS % 32 == 0, "tile shape");
};

// One pipeline stage of input rows.  No bounds: the ring is zero-initialised and only ever walked
// backwards, rows outside a tile's span meet zero taps.
template <int CH>
__device__ __forceinline__ void rs_load_rows(double (&x)[RS_G][CH], const double *col, long &row, long ring_len, int C)
{
#pragma unroll
	for (int j = 0; j < RS_G; ++j) {
		const double *p = col + row * C;
		if (CH == 4) {
			const double2 a = *reinterpret_cast<const double2 *>(p), b = *reinterpret_cast<const double2 *>(p + 2);
			x[j][0] = a.x; x[j][1 % CH] = a.y; x[j][2 % CH] = b.x; x[j][3 % CH] = b.y;
		}
		else if (CH == 2) {
			const double2 a = *reinterpret_cast<const double2 *>(p);
			x[j][0] = a.x; x[j][1 % CH] = a.y;
		}
		else x[j][0] = p[0];
		row = (row == 0) ? ring_len - 1 : row - 1;
	}
}

// Stores of 2 or 4 adjacent output channels.  `out16` (uniform: the caller's `out` is 16-byte aligned, and every
// store address is `out` plus a multiple of 16 bytes) picks 128-bit stores; without it the same values go out as
// 64-bit stores, so that an `out` that is only 8-byte aligned (legal for double) takes the same bits.
__device__ __forceinline__ void rs_store2(double *o, bool out16, double a, double b)
{
	if (out16) *reinterpret_cast<double2 *>(o) = make_double2(a, b);
	else { o[0] = a; o[1] = b; }
}

__device__ __forceinline__ void rs_store4(double *o, bool out16, double a, double b, double c, double d)
{
	rs_store2(o, out16, a, b);
	rs_store2(o + 2, out16, c, d);
}

// The input rows the tile of Q outputs from q0 reads: down from i_top, the window end of its last output (q clamped: a
// partial last tile repeats the last frame's work and does not store it), k_end rows to the window start of its first.
struct RsSpan { long i_top; int k_end; };
template <int Q> __device__ __forceinline__ RsSpan rs_span(long q0, long m0, long n_out, int n, int d, int in_len)
{
	const long q_last = (q0 + Q - 1 < n_out) ? q0 + Q - 1 : n_out - 1;
	const long i_top = ((m0 + q_last) * d) / n;
	long i_bot = ((m0 + q0) * d) / n - in_len + 1;
	if (i_bot < 0) i_bot = 0;   // rows before the stream start are zero
	return { i_top, (int) (i_top - i_bot + 1) };
}

// Where in G the taps of output q start: its phase's row, at the tap it applies to input row i_top (the index may be
// <= 0: left pad of G's rows); q clamped like the span's last output.
__device__ __forceinline__ long rs_tap_row(long q, long m0, long n_out, int n, int d, int g_stride, int pad, long i_top)
{
	if (q >= n_out) q = n_out - 1;
	const long md = (m0 + q) * d, ih = md / n;
	return (md - ih * n) * g_stride + pad + (ih - i_top);
}

template <int R, int CH, int WARPS, int MINB>
__global__ void __launch_bounds__(32 * WARPS, MINB) k_rs_poly(const double *__restrict__ ring, long ring_len, int C, const double *__restrict__ G,
                                                              int g_stride, int pad, int n, int d, int in_len, long m0, long n_out, double *__restrict__ out,
                                                              bool out16)
{
	using Cfg = RsCfg<R, CH, WARPS>;
	constexpr int Q = Cfg::Q, LD = Cfg::LD, ROWS = Cfg::ROWS;
	__shared__ __align__(16) double S[ROWS * LD];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int c0 = (blockIdx.y * 32 + lane) * CH;
	const long q0 = (long) blockIdx.x * Q;
	const auto [i_top, k_end] = rs_span<Q>(q0, m0, n_out, n, d, in_len);
	double acc[R][CH];
#pragma unroll
	for (int r = 0; r < R; ++r)
#pragma unroll
		for (int h = 0; h < CH; ++h) acc[r][h] = 0.0;
	const bool act = c0 < C;
	const double *col = ring + (act ? c0 : 0);   // lanes past the last channel compute on channel 0 and do not store
	long row = i_top % ring_len;   // next row to LOAD (runs one stage ahead of the multiplication)

	double xn[RS_G][CH];
	rs_load_rows<CH>(xn, col, row, ring_len, C);
	for (int kk = 0; kk < k_end; kk += ROWS) {
		// taps of the next ROWS rows: warp w gathers columns w, w + WARPS, ...; a lane reads consecutive taps of
		// one row of G (coalesced) and stores them down a column of S
		if (kk > 0) __syncthreads();
		for (int fr = warp; fr < Q; fr += WARPS) {
			const double *gsrc = G + rs_tap_row(q0 + fr, m0, n_out, n, d, g_stride, pad, i_top) + kk;   // tap for row i_top - kk
#pragma unroll
			for (int k = lane; k < ROWS; k += 32) S[k * LD + fr] = (kk + k < k_end) ? __ldg(gsrc + k) : 0.0;
		}
		__syncthreads();
		const int stages = (k_end - kk < ROWS) ? (k_end - kk + RS_G - 1) / RS_G : ROWS / RS_G;
		for (int sg = 0; sg < stages; ++sg) {
			double x[RS_G][CH];
#pragma unroll
			for (int j = 0; j < RS_G; ++j)
#pragma unroll
				for (int h = 0; h < CH; ++h) x[j][h] = xn[j][h];
			rs_load_rows<CH>(xn, col, row, ring_len, C);
#pragma unroll
			for (int j = 0; j < RS_G; ++j) {
				const double2 *w2 = reinterpret_cast<const double2 *>(&S[(sg * RS_G + j) * LD + warp * R]);
#pragma unroll
				for (int r = 0; r < R; r += 2) {
					const double2 w = w2[r / 2];
#pragma unroll
					for (int h = 0; h < CH; ++h) {
						acc[r][h] = fma(w.x, x[j][h], acc[r][h]);
						acc[r + 1][h] = fma(w.y, x[j][h], acc[r + 1][h]);
					}
				}
			}
		}
	}
	if (!act) return;
#pragma unroll
	for (int r = 0; r < R; ++r) {
		const long q = q0 + warp * R + r;
		if (q >= n_out) break;
		double *o = out + q * C + c0;
		if (CH == 4) rs_store4(o, out16, acc[r][0], acc[r][1 % CH], acc[r][2 % CH], acc[r][3 % CH]);
		else if (CH == 2) rs_store2(o, out16, acc[r][0], acc[r][1 % CH]);
		else o[0] = acc[r][0];
	}
}

// ---- the same sum on the FP64 tensor cores --------------------------------------------------------
// Y[q][c] = sum_k S[k][q] X[k][c] is a GEMM (M = output frames, N = channels, K = input rows) whose A operand
// is the tap tile above and whose B operand is the input ring itself.  mma.sync m8n8k4 f64 (DMMA; twice the DFMA
// rate on H100 by the data sheet, scripts/micro/dmma_probe.cu measures both) takes its
// operands as fragments -- one A and one B double per lane feed 256 FMAs -- so the L1/LSU traffic per flop
// drops by about 4x against the register-tiled FMA loop, which is what bounded that loop.
//   warp tile: 32 outputs (MT = 4 m-tiles) x 32 channels (NT = 4 n-tiles), 32 accumulator doubles per lane;
//   CTA: WARPS warps side by side along the channels, all on the same 32 outputs (one tap tile per CTA, the
//   input rows are read exactly once per CTA);
//   A fragment (m = lane/4, k = lane%4) = S[k0 + lane%4][8 mt + lane/4]: row stride 40 doubles puts the four
//   rows of a fragment on two disjoint halves of the banks (2 wavefronts for 256 bytes);
//   B fragment (k = lane%4, n = lane/4): n-tile j, column n is channel c0 + 4 n + j, so a lane's four
//   fragments are 4 adjacent channels of ONE input row -- two 128-bit loads, a warp load instruction covers
//   4 rows x 256 contiguous bytes -- and a lane's 8 results per output frame are 8 adjacent channels.
// Needs channels % 4 == 0 (16-byte aligned rows); other shapes use the FMA kernel above.
__device__ __forceinline__ void dmma884(double (&c)[2], double a, double b)
{
	asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

constexpr int RSM_Q = 32, RSM_LD = 40, RSM_ROWS = 128, RSM_MT = 4, RSM_NT = 4;

// B operand of one step: 4 adjacent channels of ring row `row` as two 128-bit loads; the row then moves down the 4
// rows of the step (k = 4), wrapping around the ring
__device__ __forceinline__ void rs_load_b(double (&b)[RSM_NT], const double *col, long &row, long ring_len, int C)
{
	const double *p = col + row * C;
	const double2 u = *reinterpret_cast<const double2 *>(p), v = *reinterpret_cast<const double2 *>(p + 2);
	b[0] = u.x; b[1] = u.y; b[2] = v.x; b[3] = v.y;
	row -= 4;
	if (row < 0) row += ring_len;
}
// A fragments of step st of a tap tile S (rows 4 st .. 4 st + 3), then the step's MT x NT DMMAs.  The kernels hold the
// fragments: with them inside one helper, ptxas assigns k_rs_mma's registers differently.
__device__ __forceinline__ void rs_load_a(double (&a)[RSM_MT], const double *S, int st, int g, int t)
{
#pragma unroll
	for (int mt = 0; mt < RSM_MT; ++mt) a[mt] = S[(4 * st + t) * RSM_LD + 8 * mt + g];
}
__device__ __forceinline__ void rs_dmma_step(double (&acc)[RSM_MT][RSM_NT][2], const double (&a)[RSM_MT], const double (&b)[RSM_NT])
{
#pragma unroll
	for (int mt = 0; mt < RSM_MT; ++mt)
#pragma unroll
		for (int j = 0; j < RSM_NT; ++j) dmma884(acc[mt][j], a[mt], b[j]);
}
// D fragment: row lane/4, columns 2 t and 2 t + 1 of n-tile j = channels c0w + 8 t + j and c0w + 8 t + 4 + j
__device__ __forceinline__ void rs_dmma_store(const double (&acc)[RSM_MT][RSM_NT][2], double *out, bool out16, long q0, long n_out, int C, int c0w, int g, int t)
{
	const int ch = c0w + 8 * t;
#pragma unroll
	for (int mt = 0; mt < RSM_MT; ++mt) {
		const long q = q0 + 8 * mt + g;
		if (q >= n_out) continue;
		double *o = out + q * C + ch;
		if (ch < C) rs_store4(o, out16, acc[mt][0][0], acc[mt][1][0], acc[mt][2][0], acc[mt][3][0]);
		if (ch + 4 < C) rs_store4(o + 4, out16, acc[mt][0][1], acc[mt][1][1], acc[mt][2][1], acc[mt][3][1]);
	}
}

template <int WARPS>
__global__ void __launch_bounds__(32 * WARPS, (WARPS == 4) ? 4 : 1) k_rs_mma(const double *__restrict__ ring, long ring_len, int C, const double *__restrict__ G,
                                                       int g_stride, int pad, int n, int d, int in_len, long m0, long n_out, double *__restrict__ out,
                                                       bool out16)
{
	constexpr int MT = RSM_MT, NT = RSM_NT, Q = RSM_Q, LD = RSM_LD, ROWS = RSM_ROWS;
	__shared__ __align__(16) double S[ROWS * LD];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
	const int c0w = (blockIdx.y * WARPS + warp) * 32;
	const long q0 = (long) blockIdx.x * Q;
	const auto [i_top, k_end] = rs_span<Q>(q0, m0, n_out, n, d, in_len);
	double acc[MT][NT][2];
#pragma unroll
	for (int mt = 0; mt < MT; ++mt)
#pragma unroll
		for (int j = 0; j < NT; ++j) acc[mt][j][0] = acc[mt][j][1] = 0.0;
	// B operand: 4 adjacent channels of row i_top - (4 step + t); lanes past the last channel read channel 0
	const int cl = c0w + 4 * g;
	const double *col = ring + ((cl < C) ? cl : 0);
	long row = (i_top - t) % ring_len;
	if (row < 0) row += ring_len;
	double bn[NT];
	rs_load_b(bn, col, row, ring_len, C);
	for (int kk = 0; kk < k_end; kk += ROWS) {
		if (kk > 0) __syncthreads();
		// gather: this lane fills columns g, g + 8, g + 16, g + 24 of S, rows k = 4 kg + t (the pointers are
		// rebuilt per chunk rather than kept in registers through the multiply loop)
		const double *gs[MT];
#pragma unroll
		for (int m = 0; m < MT; ++m) gs[m] = G + rs_tap_row(q0 + g + 8 * m, m0, n_out, n, d, g_stride, pad, i_top) + kk;   // tap of row i_top - kk
		for (int kg = warp; kg < ROWS / 4; kg += WARPS) {
			const int k = 4 * kg + t;
			const bool in = kk + k < k_end;
#pragma unroll
			for (int m = 0; m < MT; ++m) S[k * LD + g + 8 * m] = in ? __ldg(gs[m] + k) : 0.0;
		}
		__syncthreads();
		const int left = k_end - kk;
		const int steps = (left < ROWS) ? (left + 3) / 4 : ROWS / 4;
		for (int st = 0; st < steps; ++st) {
			double b[NT];
#pragma unroll
			for (int j = 0; j < NT; ++j) b[j] = bn[j];
			rs_load_b(bn, col, row, ring_len, C);
			double a[MT];
			rs_load_a(a, S, st, g, t);
			rs_dmma_step(acc, a, b);
		}
	}
	rs_dmma_store(acc, out, out16, q0, n_out, C, c0w, g, t);
}

// The same kernel with the tap tile double-buffered: the gather of chunk k+1 (cp.async, 8 bytes each, straight into
// the other half of S -- no registers, zero fill past the last row) is in flight while the DMMAs of chunk k run, one
// barrier per chunk instead of a gather phase in which the CTA's four warps issue no DMMA at all.  Chunks of 64 rows: the two halves together are the 40 KB of
// the single-buffered form, four CTAs per SM as before.
constexpr int RSM2_ROWS = 64;

__device__ __forceinline__ void cp_async8(double *smem_dst, const double *gsrc, bool valid)
{
	const unsigned d = (unsigned) __cvta_generic_to_shared(smem_dst);
	const int nbytes = valid ? 8 : 0;   // 0: nothing is read, 8 zero bytes are written
	asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(d), "l"(gsrc), "r"(nbytes) : "memory");
}

// DEPTH: steps the B rows (global loads of the input ring) are requested ahead of their use (at one step ahead the
// single-buffered form spends much of its time waiting for them)
template <int WARPS, int MINB, int DEPTH>
__global__ void __launch_bounds__(32 * WARPS, MINB) k_rs_mma2(const double *__restrict__ ring, long ring_len, int C, const double *__restrict__ G,
                                                        int g_stride, int pad, int n, int d, int in_len, long m0, long n_out, double *__restrict__ out,
                                                        bool out16)
{
	constexpr int MT = RSM_MT, NT = RSM_NT, Q = RSM_Q, LD = RSM_LD, ROWS = RSM2_ROWS;
	__shared__ __align__(16) double S[2][ROWS * LD];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
	const int c0w = (blockIdx.y * WARPS + warp) * 32;
	const long q0 = (long) blockIdx.x * Q;
	const RsSpan span = rs_span<Q>(q0, m0, n_out, n, d, in_len);   // not bound to names: gather() captures k_end
	const long i_top = span.i_top; const int k_end = span.k_end;
	double acc[MT][NT][2];
#pragma unroll
	for (int mt = 0; mt < MT; ++mt)
#pragma unroll
		for (int j = 0; j < NT; ++j) acc[mt][j][0] = acc[mt][j][1] = 0.0;
	// this lane fills columns g, g + 8, g + 16, g + 24 of S, rows k = 4 kg + t: tap of row i_top - k of the output
	// frame's phase
	long goff[MT];
#pragma unroll
	for (int m = 0; m < MT; ++m) goff[m] = rs_tap_row(q0 + g + 8 * m, m0, n_out, n, d, g_stride, pad, i_top);
	auto gather = [&](int kk, double *Sb) {
		for (int kg = warp; kg < ROWS / 4; kg += WARPS) {
			const int k = 4 * kg + t;
			const bool in = kk + k < k_end;
#pragma unroll
			for (int m = 0; m < MT; ++m) cp_async8(&Sb[k * LD + g + 8 * m], G + (in ? goff[m] + kk + k : 0), in);
		}
		asm volatile("cp.async.commit_group;" ::: "memory");
	};
	gather(0, S[0]);
	// B operand: 4 adjacent channels of row i_top - (4 step + t); lanes past the last channel read channel 0
	const int cl = c0w + 4 * g;
	const double *col = ring + ((cl < C) ? cl : 0);
	long row = (i_top - t) % ring_len;
	if (row < 0) row += ring_len;
	double bq[DEPTH][NT];
#pragma unroll
	for (int dd = 0; dd < DEPTH; ++dd) rs_load_b(bq[dd], col, row, ring_len, C);
	asm volatile("cp.async.wait_group 0;" ::: "memory");
	__syncthreads();
	int cur = 0;
	for (int kk = 0; kk < k_end; kk += ROWS) {
		if (kk + ROWS < k_end) gather(kk + ROWS, S[cur ^ 1]);   // nobody reads that half any more (barrier below)
		const int left = k_end - kk;
		const int steps = (left < ROWS) ? (left + 3) / 4 : ROWS / 4;
		for (int st = 0; st < steps; ++st) {
			double b[NT];
#pragma unroll
			for (int j = 0; j < NT; ++j) b[j] = bq[0][j];
#pragma unroll
			for (int dd = 0; dd + 1 < DEPTH; ++dd)
#pragma unroll
				for (int j = 0; j < NT; ++j) bq[dd][j] = bq[dd + 1][j];
			rs_load_b(bq[DEPTH - 1], col, row, ring_len, C);
			double a[MT];
			rs_load_a(a, S[cur], st, g, t);
			rs_dmma_step(acc, a, b);
		}
		asm volatile("cp.async.wait_group 0;" ::: "memory");
		__syncthreads();   // the next half is complete and visible; this half is free
		cur ^= 1;
	}
	rs_dmma_store(acc, out, out16, q0, n_out, C, c0w, g, t);
}

using RsKernel = void (*)(const double *, long, int, const double *, int, int, int, int, int, long, long, double *, bool);
// The instantiation that runs a launch, its template arguments read from rs_variant() (resample_plan.h), so that
// describe() reports what ran.  The FMA tiles have fixed warps: rs_instance<T, W> is the same kernel for every W.
template <int T, int W> static RsKernel rs_instance()
{
	constexpr RsLaunch v = rs_variant(T, W);
	static_assert((T <= 3) ? v.Q % v.warps == 0 && v.channels % 32 == 0 : v.Q == RSM_Q && v.channels == 32 * W, "variant's tile");
	static_assert(T != 4 || v.minb == ((W == 4) ? 4 : 1), "k_rs_mma's launch bounds");
	if constexpr (T <= 3) return k_rs_poly<v.Q / v.warps, v.channels / 32, v.warps, v.minb>;
	else if constexpr (T == 4) return k_rs_mma<W>;
	else return k_rs_mma2<W, v.minb, v.depth>;
}
template <int T> static RsKernel rs_tile_kernel(int w) { return (w == 4) ? rs_instance<T, 4>() : (w == 2) ? rs_instance<T, 2>() : rs_instance<T, 1>(); }
static RsKernel (*const rs_kernel[8])(int warps) = { nullptr, rs_tile_kernel<1>, rs_tile_kernel<2>, rs_tile_kernel<3>, rs_tile_kernel<4>,
                                                     rs_tile_kernel<5>, rs_tile_kernel<6>, rs_tile_kernel<7> };   // by tile

// move the live rows of the input ring into a bigger ring (absolute frame a lives at a % len)
__global__ void k_rs_ring_grow(const double *old_ring, long old_len, double *new_ring, long new_len, int C, long a0, long rows)
{
	const long idx = (long) blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= rows * C) return;
	const long a = a0 + idx / C;
	const int c = (int) (idx % C);
	new_ring[(a % new_len) * C + c] = old_ring[(a % old_len) * C + c];
}

struct ResampleOp : Op {
	RsPacing pace;
	const ResampleParams &p = pace.p;
	double *d_G = nullptr, *d_ring = nullptr;
	int g_stride = 0, g_pad = 0;         // tap rows: [pad zeros | in_len taps | pad zeros]
	long ring_len = 0, total_in = 0;   // total_in: frames appended since reset
	int force_tile = 0;         // DSP_B200_RS_TILE (resample_plan.h), read when the operator is made
	// the last launch, for describe(), and the alignment of its output in bytes (16: 128-bit stores, 8: 64-bit stores)
	RsLaunch last; int last_out_align = 0;

	const char *name() const override { return "resample"; }

	std::string describe() const override
	{
		char buf[384];
		snprintf(buf, sizeof(buf), "{\"op\":\"resample\",\"n\":%d,\"d\":%d,\"in_len\":%d,\"out_len\":%d,\"out_delay\":%d,\"ring_len\":%ld,"
		         "\"force_tile\":%d,\"kernel\":\"%s\",\"tile\":%d,\"warps\":%d,\"depth\":%d,\"out_align\":%d}",
		         p.n, p.d, p.in_len, p.out_len, p.out_delay, ring_len, force_tile, last.kernel, last.tile, last.warps, last.depth, last_out_align);
		return buf;
	}
	~ResampleOp() override { dev_free(d_G); dev_free(d_ring); }

	long max_out_frames(long in_frames) const override { return pace.max_out_frames(in_frames); }

	void reset(cudaStream_t st) override
	{
		pace.reset();
		total_in = 0;
		if (d_ring) cudaMemsetAsync(d_ring, 0, (size_t) ring_len * channels * sizeof(double), st);
	}

	int ensure_ring(long frames, cudaStream_t st)
	{
		const long need = 3L * p.in_len + frames + 64;
		if (ring_len >= need) return 0;
		const long new_len = 3L * p.in_len + 2 * frames + 64;
		double *nr = dev_alloc<double>((size_t) new_len * channels, true);
		if (!nr) return -1;
		if (d_ring) {
			const long rows = (total_in < ring_len) ? total_in : ring_len;
			if (rows > 0)
				LAUNCH(k_rs_ring_grow, ceil_div(rows * channels, 256), 256, 0, st, d_ring, ring_len, nr, new_len, channels, total_in - rows, rows);
			CUDA_TRY(cudaStreamSynchronize(st), return -1);
			dev_free(d_ring);
		}
		d_ring = nr;
		ring_len = new_len;
		return 0;
	}

	long run(long frames, const double *in, double *out, cudaStream_t st) override
	{
		if (frames <= 0) return 0;
		const int C = channels, sms = sm_count();
		if (sms < 1 || ensure_ring(frames, st)) return -1;
		// append the new rows (at most one wrap)
		{
			const long w = total_in % ring_len;
			const long first = (frames < ring_len - w) ? frames : ring_len - w;
			CUDA_TRY(cudaMemcpyAsync(d_ring + w * C, in, (size_t) first * C * sizeof(double), cudaMemcpyDeviceToDevice, st), return -1);
			if (first < frames)
				CUDA_TRY(cudaMemcpyAsync(d_ring, in + first * C, (size_t) (frames - first) * C * sizeof(double), cudaMemcpyDeviceToDevice, st), return -1);
			total_in += frames;
		}
		const RsCall call = pace.run(frames);   // resample_effect_run()'s pacing
		if (call.frames < 0) set_error("resample: pacing stalled (in_buf_pos=%d out_buf_pos=%d)", pace.in_buf_pos, pace.out_buf_pos);
		if (call.frames <= 0) return call.frames;   // -1 when stalled
		ProfScope prof("resample", st);
		last = rs_launch(C, call.frames, sms, force_tile);
		// the stores into the caller's rows: 128-bit when `out` allows it (a row offset is a multiple of 16 bytes
		// wherever a kernel stores pairs), else 64-bit -- the same values either way
		const bool out16 = (reinterpret_cast<uintptr_t>(out) & 15) == 0;
		last_out_align = out16 ? 16 : 8;
		const dim3 grid((unsigned) ceil_div(call.frames, last.Q), (unsigned) ceil_div(C, last.channels));
		LAUNCH(rs_kernel[last.tile](last.warps), grid, 32 * last.warps, 0, st, d_ring, ring_len, C, d_G, g_stride, g_pad, p.n, p.d, p.in_len, call.first, call.frames,
		       out, out16);
		return call.frames;
	}

	// resample.c:163-188
	long drain2(long frames, double *zeros, double *out, cudaStream_t st) override
	{
		if (pace.drain_dry()) return -1;
		CUDA_TRY(cudaMemsetAsync(zeros, 0, (size_t) frames * channels * sizeof(double), st), return -2);
		const long produced = run(frames, zeros, out, st);
		return (produced < 0) ? -2 : pace.drain_trim(produced);
	}
};

Op *make_resample_op(int slab_channels, int fs_in, int fs_out, double bandwidth, cudaStream_t st)
{
	std::unique_ptr<ResampleOp> op(new ResampleOp());
	op->channels = slab_channels;
	op->fs_in = fs_in;
	op->fs_out = fs_out;
	op->inplace_ok = false;
	op->force_tile = getenv("DSP_B200_RS_TILE") ? atoi(getenv("DSP_B200_RS_TILE")) : 0;
	if (resample_params_or_error(fs_in, fs_out, bandwidth, &op->pace.p)) return nullptr;
	const ResampleParams &p = op->p;

	// windowed sinc, resample.c:361-364 (host libm, like the reference)
	std::vector<double> sinc((size_t) p.m_os + 1, 0.0);
	for (int i = 1; i < p.m_os; ++i) {
		const double x = (i * 2 - p.m_os) / 2.0;
		const double s = (fabs(x) < 1e-9) ? p.fc_os : sin(M_PI * p.fc_os * x) / (M_PI * x);
		sinc[i] = s * albrecht9((double) i / p.m_os);
	}
	double *d_sinc = dev_alloc<double>(sinc.size(), false);
	double2 *d_S = dev_alloc<double2>((size_t) p.sinc_len + 1, false);
	// Q consecutive outputs span at most (Q-1) d/n + 1 input rows more than one output does
	op->g_pad = (int) (((long) (RS_QMAX - 1) * p.d) / p.n + 2);
	op->g_stride = p.in_len + 2 * op->g_pad;
	op->d_G = dev_alloc<double>((size_t) p.n * op->g_stride, true);
	if (!d_sinc || !d_S || !op->d_G) return nullptr;
	CUDA_TRY(cudaMemcpyAsync(d_sinc, sinc.data(), sinc.size() * sizeof(double), cudaMemcpyHostToDevice, st), return nullptr);
	LAUNCH(k_rs_sinc_dft, ceil_div(p.sinc_len + 1, 128), 128, 0, st, d_sinc, p.m_os, p.sinc_len, d_S);
	LAUNCH(k_rs_table, ceil_div((long) p.n * p.in_len, 128), 128, 0, st, d_S, p.sinc_len, p.n, p.in_len, op->d_G, op->g_stride, op->g_pad);
	CUDA_TRY(cudaStreamSynchronize(st), return nullptr);
	dev_free(d_sinc);
	dev_free(d_S);
	return op.release();
}

}  // namespace dspb200
