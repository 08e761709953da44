// fir_pipe.cuh -- K2's block kernel as ONE persistent, warp-specialised pipeline per block (single-level plans).
//
// One CTA per SM.  For block j the launch does ALL the device work of the block:
//   (a) per channel s (s = blockIdx.x, blockIdx.x + gridDim.x, ...):
//         S = X_j H_0 + sum_{1 <= p < pf} X_{j-p} H_p + V_j        (reference: fft_part_group_compute, fir_p.c:64-103)
//         y = IRFFT(S)[0:B) + carry,  carry' = IRFFT(S)[B:2B)
//   (b) the time-batched tail for a QUARTER of the channels (those with s % 4 == j % 4):
//         V_{j+2+t} = sum_{p >= pf} X_{j+2+t-p} H_p,  t = 0..3      -- only blocks <= j-1 are involved, so nothing in
//       this launch depends on anything else in it; every FDL and filter row is streamed once for four outputs (the
//       filter rows slide through a register window).  Spreading the batch over the channels' residues makes every
//       launch the same work: no side streams, no events, one kernel per block.
// Three kinds of warps that only meet at mbarriers:
//   producer (1 warp, one lane)   the scheduler: streams row chunks from HBM into a ring of shared-memory stages with
//                                 cp.async.bulk (TMA bulk copies, completion counted in bytes on the stage's "full"
//                                 mbarrier) and tags every stage with a command word.  It issues the stages of (a) as
//                                 soon as the spectrum buffer `sbuf` is free for the channel and fills all other time
//                                 with its share of the work items of (b) -- the HBM stream never waits for a transform.
//   MAC warps (4)                 execute the command of each stage: complex multiply-accumulate of 256 bins (2 per
//                                 lane) into registers, sums of (a) dropped into `sbuf`, sums of (b) stored to V
//   transform team (N/16 threads) reads the caller's interleaved block, forward FFT in shared memory, spectrum to the
//                                 FDL, S = sbuf + X_j H_0 for the bin pairs it owns, inverse FFT in place,
//                                 overlap-add, writes the caller's interleaved result.  It is latency-bound (two
//                                 warps per scheduler) -- and that no longer matters: the kernel's duration is set by
//                                 the byte stream, which runs beside it at the speed of the HBM.
// sbuf is handed back and forth by two mbarriers (s_full: MAC -> team, s_empty: team -> producer); the team synchronises
// itself with a named barrier.
#pragma once
#include "common.cuh"
#include "fft.cuh"
#include "fir_plan.h"
#include "fir_tile.cuh"
#include <cstdint>

namespace dspb200 {

template <int N>
struct PipeCfg {
	static constexpr int TF = N / 16;                 // transform team (one FFT)
	static constexpr int MAC_WARPS = 4;               // 8 + 4 + 1 warps: at most 4 warps per SM sub-partition, 128 registers each
	static constexpr int TM = MAC_WARPS * 32;
	static constexpr int THREADS = TF + TM + 32;      // + producer warp
	static constexpr int CHUNK = 256;                 // bins per stage
	static constexpr int NCHUNK = N / CHUNK;
	static constexpr int PER = CHUNK / TM;            // bins per MAC lane and stage
	static constexpr int SLOTS = 2;                   // (X chunk | H chunk) pairs per stage: one barrier round trip per two rows
	static constexpr int NS = (N >= 4096) ? 5 : 8;    // ring stages (16 KB each)
	static constexpr size_t STAGE_BYTES = SLOTS * 2 * (size_t) CHUNK * sizeof(double2);
	static constexpr size_t FBUF = (size_t) FftCfg<N>::STRIDE * sizeof(double2);
	static constexpr size_t SBUF = (size_t) N * sizeof(double2);
	static constexpr size_t CMDS = (size_t) NS * sizeof(int4);
	static constexpr size_t SMEM = FBUF + SBUF + NS * STAGE_BYTES + CMDS + (2 * NS + 2) * sizeof(uint64_t);
	static_assert(TF % 32 == 0 && N % CHUNK == 0 && CHUNK % TM == 0, "shape");
};

struct PipeArgs {
	const double *xin;       // caller's interleaved block
	long xin_stride;
	const int *xin_map;      // channel of selected channel s (NULL: s)
	double *yout;
	long yout_stride;
	const int *yout_map;
	double2 *fdl;            // [s][fdl_rows][N]
	long fdl_ch_stride;
	int fdl_rows, slot;      // slot = row of block j
	const double2 *H;        // [s or 0][P][N]
	long h_ch_stride;        // 0: shared filter
	int P;                   // partitions of the filter
	int pf;                  // partitions summed in (a): 0 .. pf-1
	double2 *V;              // [v_slots][n_ch][N]: batched spectra, slot = block index % v_slots (NULL: no batching, pf == P)
	int v_slots;
	long blk;                // j
	double *carry;           // [s][N]
	const double2 *tw, *ptw;
	int n_ch;
	int evict_first;         // streaming operands are read once per block: keep them from displacing the rest of L2
	int fake_io;             // MEASUREMENT ONLY (DSP_B200_FIR_PIPE_FAKEIO): contiguous block I/O (wrong results) to time the kernel without the strided accesses
	int no_batch_items;      // MEASUREMENT ONLY: skip (b)
	long long *stats;        // MEASUREMENT ONLY: [gridDim.x][8] cycle counters (NULL: off)
};

// stage commands (producer -> MAC warps)
enum {
	PC_SZERO = 1,      // (a): clear the sum
	PC_SMAC = 2,       //      sum += X . H
	PC_SADDV = 4,      //      sum += the chunk in the X slot (V_j)
	PC_SSTORE = 8,     //      sum -> sbuf[chunk]
	PC_SFULL = 16,     //      last chunk of the channel: sbuf is complete
	PC_BINIT = 32,     // (b): clear the four sums and the window; window[3] = chunk in the H slot (PC_BHASH)
	PC_BSTEP = 64,     //      sums[t] += X . window[t]; window slides; window[3] = chunk in the H slot (PC_BHASH) or 0
	PC_BHASH = 128,
	PC_BSTORE = 256,   //      sums -> V[(j + 2 + t) % v_slots][s][chunk]
	PC_EXIT = 512
};

// Register cap: the register file is split over the SM's four sub-partitions (16384 each) and a CTA's warps are dealt
// round-robin: 13 warps = at most 4 per sub-partition = 128 registers per thread (a 17-warp layout with 8 MAC warps
// would have to fit 5 x 32 x R <= 16384, i.e. 96 registers, which the transform team cannot live with).
#ifndef FIR_PIPE_MAXNREG
#define FIR_PIPE_MAXNREG 128
#endif

template <int N>
__global__ void __maxnreg__(FIR_PIPE_MAXNREG) k_fir_pipe(PipeArgs a)
{
	using Cfg = PipeCfg<N>;
	constexpr int T = Cfg::TF, CHUNK = Cfg::CHUNK, NS = Cfg::NS, PER = Cfg::PER, TM = Cfg::TM, TB = PIPE_TB;
	using TeamSync = NamedSync<1, T>;
	extern __shared__ __align__(128) unsigned char smem_raw[];
	double2 *fbuf = reinterpret_cast<double2 *>(smem_raw);
	double2 *sbuf = reinterpret_cast<double2 *>(smem_raw + Cfg::FBUF);
	double2 *ring = reinterpret_cast<double2 *>(smem_raw + Cfg::FBUF + Cfg::SBUF);
	int4 *cmds = reinterpret_cast<int4 *>(smem_raw + Cfg::FBUF + Cfg::SBUF + NS * Cfg::STAGE_BYTES);
	uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + Cfg::FBUF + Cfg::SBUF + NS * Cfg::STAGE_BYTES + Cfg::CMDS);
	uint64_t *full = bars, *empty = bars + NS, *s_full = bars + 2 * NS, *s_empty = bars + 2 * NS + 1;

	if (threadIdx.x == 0) {
		for (int i = 0; i < NS; ++i) {
			mbar_init(&full[i], 1);                  // the producer's arrive.expect_tx; the copies complete the bytes
			mbar_init(&empty[i], Cfg::MAC_WARPS);    // one arrival per MAC warp
		}
		mbar_init(s_full, Cfg::MAC_WARPS);
		mbar_init(s_empty, T / 32);                  // one arrival per team warp
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();   // the only CTA-wide barrier: from here on the roles meet at mbarriers

	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const bool stats_on = a.stats != nullptr;
	long long t_begin = stats_on ? clock64() : 0, t_wait = 0;

	if (warp < T / 32) {
		// ------------------------------------------------------------------------------------------
		// transform team
		// ------------------------------------------------------------------------------------------
		const int t = threadIdx.x;
		double2 *buf = fbuf;
		int it = 0;
		for (int s = blockIdx.x; s < a.n_ch; s += gridDim.x, ++it) {
			double2 *fdl = a.fdl + (long) s * a.fdl_ch_stride;
			const double2 *H0 = a.H + (long) s * a.h_ch_stride;
			double2 *X = fdl + (long) a.slot * N;
			double2 *carry = reinterpret_cast<double2 *>(a.carry + (long) s * N);
			{
				// frames 2n, 2n+1 of this channel (the CTAs next door read the rest of each sector at about the same time)
				const double *xc = a.fake_io ? a.xin + (long) s * N : a.xin + (a.xin_map ? a.xin_map[s] : s);
				const long xs = a.fake_io ? 1 : a.xin_stride;
				double2 v[8];
				read_frame_pairs<T>(v, xc, xs, t);   // plain loads: the call may be in place
				// what the later phases read with plain loads: on its way to L2 while the first transform runs
				prefetch_rows(H0, (long) N * sizeof(double2), t, T);
				prefetch_rows(carry, (long) N * sizeof(double), t, T);
				fill_buf<N, T>(buf, v, t);
			}
			TeamSync::sync();
			fft_forward_smem<N, TeamSync>(buf, a.ptw, t);
			double2 w[8];
#pragma unroll
			for (int i = 0; i < 8; ++i) w[i] = __ldg(&a.tw[t + i * T]);
			// (1) real split: X[k], X[N-k] to the FDL and, in place of Z, to shared memory.
			//     Thread t owns the pairs k = t + i T; thread 0 also owns k = 0 (packed DC/Nyquist) and k = N/2.
#pragma unroll
			for (int i = 0; i < 8; ++i)
				rfft_split<N>(buf, t + i * T, w[i], [&](int k, int n, double2 xk, double2 xn) {
					X[k] = xk; X[n] = xn;
					buf[spad(k)] = xk; buf[spad(n)] = xn;
				});
			// (2) S = X_j H_0 + (what the MAC warps summed for this channel), inverse merge into shared memory
			{
				const long long t0 = stats_on ? clock64() : 0;
				mbar_wait(s_full, (unsigned) (it & 1));
				if (stats_on) t_wait += clock64() - t0;
			}
#pragma unroll
			for (int i = 0; i < 8; ++i) {
				const int k = t + i * T;
				const int n = (k == 0) ? N / 2 : N - k;
				const double2 xk = buf[spad(k)], xn = buf[spad(n)];
				const double2 hk = __ldg(&H0[k]), hn = __ldg(&H0[n]);
				double2 Sk = sbuf[k], Sn = sbuf[n];
				cmac_packed(Sk, xk, hk, k == 0);
				Sn = cmac(Sn, xn, hn);
				irfft_merge<N>(buf, k, n, Sk, Sn, w[i]);
			}
			__syncwarp();
			if (lane == 0) mbar_arrive(s_empty);   // sbuf may be refilled for the next channel
			TeamSync::sync();
			fft_forward_smem<N, TeamSync>(buf, a.ptw, t);
			// (3) overlap-add, result into the caller's block
			{
				const double scale = 1.0 / N;
				double *yc = a.fake_io ? a.yout + (long) s * N : a.yout + (a.yout_map ? a.yout_map[s] : s);
				const long ys = a.fake_io ? 1 : a.yout_stride;
				double2 c[8];
#pragma unroll
				for (int i = 0; i < 8; ++i) c[i] = carry[t + i * T];
#pragma unroll
				for (int i = 0; i < 8; ++i) {
					const int n = t + i * T;
					const double2 lo = buf[spad(n)], hi = buf[spad(n + N / 2)];
					const double2 y = ola_out(lo, scale, c[i]);
					yc[2L * n * ys] = y.x;
					yc[(2L * n + 1) * ys] = y.y;
					carry[n] = ola_scaled(hi, scale);
				}
			}
			// entry n and n + N/2 of buf are only touched by this thread between the last pass and the next
			// channel's first barrier: no barrier needed here
		}
		if (stats_on && threadIdx.x == 0) {
			a.stats[blockIdx.x * 8 + 0] = t_wait;
			a.stats[blockIdx.x * 8 + 3] = clock64() - t_begin;
		}
	}
	else if (warp < T / 32 + Cfg::MAC_WARPS) {
		// ------------------------------------------------------------------------------------------
		// MAC warps: execute the stages' commands
		// ------------------------------------------------------------------------------------------
		const int tm = threadIdx.x - T;
		int stage = 0;
		unsigned phase = 0;
		const double2 zero = make_double2(0.0, 0.0);
		double2 accS[PER], accB[TB][PER], hw[TB][PER];
		unsigned liveB = 0;   // bit u: hw[u] is a filter row of the batch window (window_mac())
#pragma unroll
		for (int i = 0; i < PER; ++i) {
			accS[i] = zero;
#pragma unroll
			for (int u = 0; u < TB; ++u) { accB[u][i] = zero; hw[u][i] = zero; }
		}
		{
			const long long t0 = stats_on ? clock64() : 0;
			mbar_wait(&full[stage], phase);
			if (stats_on) t_wait += clock64() - t0;
		}
		int4 cmd = cmds[stage];
		for (;;) {
			const int flw = cmd.x, chunk = cmd.y, s = cmd.z;
			if (flw & PC_EXIT) break;
			const bool dc = (chunk == 0 && tm == 0);   // bin 0 packs (DC, Nyquist): two real products
#pragma unroll
			for (int sl_ = 0; sl_ < Cfg::SLOTS; ++sl_) {
			const int fl = (sl_ == 0) ? (flw & 0xffff) : (flw >> 16);
			if (sl_ > 0 && fl == 0) break;
			const double2 *Xs = ring + ((size_t) stage * Cfg::SLOTS + sl_) * 2 * CHUNK, *Hs = Xs + CHUNK;
			if (fl & PC_BSTEP) {
#pragma unroll
				for (int i = 0; i < PER; ++i) {
					const double2 x = Xs[tm + i * TM];
					const double2 hn = (fl & PC_BHASH) ? Hs[tm + i * TM] : zero;
					// two calls with a constant dc, as the kernel had them (one call with dc && i == 0 compiles to other code)
					if (dc && i == 0) window_mac<TB, PER>(&accB[0][i], &hw[0][i], liveB, x, true);
					else window_mac<TB, PER>(&accB[0][i], &hw[0][i], liveB, x, false);
#pragma unroll
					for (int u = 0; u + 1 < TB; ++u) hw[u][i] = hw[u + 1][i];
					hw[TB - 1][i] = hn;
				}
				liveB = (liveB >> 1) | ((fl & PC_BHASH) ? 1u << (TB - 1) : 0u);
				if (fl & PC_BSTORE) {
#pragma unroll
					for (int u = 0; u < TB; ++u) {
						const long slot = (a.blk + 2 + u) % a.v_slots;
						double2 *Vd = a.V + (slot * a.n_ch + s) * (long) N + chunk * CHUNK;
#pragma unroll
						for (int i = 0; i < PER; ++i) Vd[tm + i * TM] = accB[u][i];
					}
				}
			}
			else if (fl & PC_SMAC) {
				double2 x[PER], h[PER];
#pragma unroll
				for (int i = 0; i < PER; ++i) { x[i] = Xs[tm + i * TM]; h[i] = Hs[tm + i * TM]; }
				if (fl & PC_SZERO) {
#pragma unroll
					for (int i = 0; i < PER; ++i) accS[i] = zero;
				}
				cmac_packed(accS[0], x[0], h[0], dc);
#pragma unroll
				for (int i = 1; i < PER; ++i) accS[i] = cmac(accS[i], x[i], h[i]);
				if (fl & PC_SSTORE) {
#pragma unroll
					for (int i = 0; i < PER; ++i) sbuf[chunk * CHUNK + tm + i * TM] = accS[i];
				}
			}
			else if (fl & (PC_SADDV | PC_SSTORE)) {
				if (fl & PC_SZERO) {
#pragma unroll
					for (int i = 0; i < PER; ++i) accS[i] = zero;
				}
				if (fl & PC_SADDV) {
#pragma unroll
					for (int i = 0; i < PER; ++i) {
						const double2 v = Xs[tm + i * TM];
						accS[i].x += v.x; accS[i].y += v.y;
					}
				}
#pragma unroll
				for (int i = 0; i < PER; ++i) sbuf[chunk * CHUNK + tm + i * TM] = accS[i];
			}
			else if (fl & PC_BINIT) {
#pragma unroll
				for (int i = 0; i < PER; ++i) {
#pragma unroll
					for (int u = 0; u < TB; ++u) { accB[u][i] = zero; hw[u][i] = zero; }
					if (fl & PC_BHASH) hw[TB - 1][i] = Hs[tm + i * TM];
				}
				liveB = (fl & PC_BHASH) ? 1u << (TB - 1) : 0u;
			}
			}
			__syncwarp();
			if (lane == 0) {
				if ((flw | (flw >> 16)) & PC_SFULL) mbar_arrive(s_full);   // after this warp's part of the last chunk is in sbuf
				mbar_arrive(&empty[stage]);
			}
			// (a warp issues in order: probing the next stage's barrier ahead of the arithmetic would only stall the
			// arithmetic behind the probe's answer -- so the wait comes here, once per two rows)
			const bool wrap = (stage + 1 == NS);
			stage = wrap ? 0 : stage + 1;
			phase ^= wrap ? 1u : 0u;
			{
				const long long t0 = stats_on ? clock64() : 0;
				mbar_wait(&full[stage], phase);
				if (stats_on) t_wait += clock64() - t0;
			}
			cmd = cmds[stage];
		}
		if (stats_on && tm == 0) {
			a.stats[blockIdx.x * 8 + 1] = t_wait;
			a.stats[blockIdx.x * 8 + 4] = clock64() - t_begin;
		}
	}
	else if (elect_one()) {
		// ------------------------------------------------------------------------------------------
		// producer / scheduler (one elected lane of the last warp)
		// ------------------------------------------------------------------------------------------
		const uint64_t pol = l2_policy_evict_first();
		const bool hint_x = a.evict_first != 0, hint_h = a.evict_first != 0 && a.h_ch_stride != 0;
		constexpr unsigned ROW_BYTES = CHUNK * sizeof(double2);
		constexpr int NCHUNK = Cfg::NCHUNK;
		const int G = (int) gridDim.x, b = (int) blockIdx.x;
		const int n_my = (b < a.n_ch) ? (a.n_ch - b + G - 1) / G : 0;   // channels of this CTA
		const bool has_v = a.V != nullptr && a.blk >= 3;                 // V_j exists (zero before block 3: not read)
		int stage = 0;
		unsigned phase = 0;
		long n_stages = 0;

		// Stages carry up to SLOTS (X chunk | H chunk) pairs of one chunk of one channel: entries are collected with
		// emit() and leave with flush() -- wait for the ring slot, tag it, start the copies.
		static_assert(Cfg::SLOTS == 2, "the pending stage is kept in scalars");
		int pn = 0, p_chunk = 0, p_s = 0, p_fl0 = 0, p_fl1 = 0;
		const double2 *p_x0 = nullptr, *p_h0 = nullptr, *p_x1 = nullptr, *p_h1 = nullptr;
		bool p_hx0 = false, p_hh0 = false, p_hx1 = false, p_hh1 = false;
		auto flush = [&]() {
			if (pn == 0) return;
			{
				const long long t0 = stats_on ? clock64() : 0;
				mbar_wait(&empty[stage], phase ^ 1);
				if (stats_on) t_wait += clock64() - t0;
			}
			if (pn < 2) { p_fl1 = 0; p_x1 = nullptr; p_h1 = nullptr; }
			const unsigned bytes = (p_x0 ? ROW_BYTES : 0) + (p_h0 ? ROW_BYTES : 0) + (p_x1 ? ROW_BYTES : 0) + (p_h1 ? ROW_BYTES : 0);
			cmds[stage] = make_int4(p_fl0 | (p_fl1 << 16), p_chunk, p_s, 0);
			if (bytes) mbar_arrive_expect_tx(&full[stage], bytes);
			else mbar_arrive(&full[stage]);   // nothing to copy (exit, or rows that do not exist)
			double2 *dst = ring + (size_t) stage * Cfg::SLOTS * 2 * CHUNK;
			if (p_x0) bulk_g2s(dst, p_x0, ROW_BYTES, &full[stage], p_hx0, pol);
			if (p_h0) bulk_g2s(dst + CHUNK, p_h0, ROW_BYTES, &full[stage], p_hh0, pol);
			if (p_x1) bulk_g2s(dst + 2 * CHUNK, p_x1, ROW_BYTES, &full[stage], p_hx1, pol);
			if (p_h1) bulk_g2s(dst + 3 * CHUNK, p_h1, ROW_BYTES, &full[stage], p_hh1, pol);
			if (++stage == NS) { stage = 0; phase ^= 1; }
			++n_stages;
			pn = 0;
		};
		auto emit = [&](int flags, int chunk, int s, const double2 *xsrc, const double2 *hsrc, bool hx, bool hh) {
			if (pn == 0) { p_fl0 = flags; p_x0 = xsrc; p_h0 = hsrc; p_hx0 = hx; p_hh0 = hh; }
			else { p_fl1 = flags; p_x1 = xsrc; p_h1 = hsrc; p_hx1 = hx; p_hh1 = hh; }
			p_chunk = chunk; p_s = s;
			if (++pn == 2) flush();
		};

		// (b): the channels s = g + TB k of this block's residue g, cut into NCHUNK items each; this CTA's share
		// is weighted by what (a) leaves it (CTAs that walk fewer channels take more items)
		long item = 0, item_end = 0, item0 = 0;
		const int g = (int) (a.blk % TB);
		const int n_g = (a.V && a.blk >= 1 && a.n_ch > g && !a.no_batch_items) ? (a.n_ch - g + TB - 1) / TB : 0;
		if (n_g > 0) {
			const long n_items = (long) n_g * NCHUNK;
			const long Ss = (long) NCHUNK * ((a.pf - 1 + (has_v ? 1 : 0) + Cfg::SLOTS - 1) / Cfg::SLOTS), Sb = (a.P - 2 + Cfg::SLOTS - 1) / Cfg::SLOTS;
			const long total = (long) a.n_ch * Ss + n_items * Sb;
			const long target = (total + G - 1) / G;
			long W = 0, Wb = 0, wb = 0;
			for (int c = 0; c < G; ++c) {
				const int nc = (c < a.n_ch) ? (a.n_ch - c + G - 1) / G : 0;
				long wgt = target - nc * Ss;
				if (wgt < 1) wgt = 1;
				if (c < b) Wb += wgt;
				if (c == b) wb = wgt;
				W += wgt;
			}
			item0 = item = n_items * Wb / W;
			item_end = n_items * (Wb + wb) / W;
		}

		auto emit_item = [&](long it_) {
			const int k = (int) (it_ / NCHUNK), c = (int) (it_ % NCHUNK);
			const int s = g + TB * k;
			const double2 *fdl = a.fdl + (long) s * a.fdl_ch_stride + c * CHUNK;
			const double2 *Hc = a.H + (long) s * a.h_ch_stride + c * CHUNK;
			// window[t] = H_{3+t} where it belongs to the batch (p >= pf): with pf = TB + 2 only t = TB-1 does
			const int p0 = a.pf;
			emit(PC_BINIT | ((p0 < a.P) ? PC_BHASH : 0), c, s, nullptr, (p0 < a.P) ? Hc + (long) p0 * N : nullptr, false, hint_h);
			// step m: X_{j+2-m} (one row further back per step, starting at block j-1) meets the window; next window row H_{m+TB}
			int sl = a.slot - 1;
			if (sl < 0) sl += a.fdl_rows;
			const double2 *hp = Hc + (long) (3 + TB) * N;
			for (int m = 3; m < a.P; ++m) {
				const bool hh = m + TB < a.P;
				emit(PC_BSTEP | (hh ? PC_BHASH : 0) | ((m == a.P - 1) ? PC_BSTORE : 0), c, s, fdl + (long) sl * N, hh ? hp : nullptr, hint_x, hint_h);
				hp += N;
				if (--sl < 0) sl += a.fdl_rows;
			}
			flush();
		};

		auto emit_channel = [&](int s) {
			const double2 *fdl = a.fdl + (long) s * a.fdl_ch_stride;
			const double2 *Hc = a.H + (long) s * a.h_ch_stride;
			const double2 *Vc = has_v ? a.V + ((a.blk % a.v_slots) * a.n_ch + s) * (long) N : nullptr;
			for (int c = 0; c < NCHUNK; ++c) {
				const int last = (c == NCHUNK - 1) ? PC_SFULL : 0;
				if (a.pf <= 1 && !Vc) { emit(PC_SZERO | PC_SSTORE | last, c, s, nullptr, nullptr, false, false); flush(); continue; }
				for (int p = 1; p < a.pf; ++p) {
					int sl = a.slot - p;
					if (sl < 0) sl += a.fdl_rows;
					int fl = PC_SMAC | (p == 1 ? PC_SZERO : 0);
					if (p == a.pf - 1 && !Vc) fl |= PC_SSTORE | last;
					emit(fl, c, s, fdl + (long) sl * N + c * CHUNK, Hc + (long) p * N + c * CHUNK, hint_x, hint_h);
				}
				if (Vc) emit(PC_SADDV | PC_SSTORE | last | (a.pf <= 1 ? PC_SZERO : 0), c, s, Vc + c * CHUNK, nullptr, hint_x, false);
				flush();   // a stage never mixes chunks
			}
		};

		int ci = 0;   // next channel of (a) to issue
		for (;;) {
			if (ci < n_my && (ci == 0 || mbar_try_wait(s_empty, (unsigned) ((ci & 1) ^ 1)))) {
				emit_channel(b + ci * G);
				++ci;
			}
			else if (item < item_end) emit_item(item++);
			else if (ci < n_my) {
				const long long t0 = stats_on ? clock64() : 0;
				mbar_wait(s_empty, (unsigned) ((ci & 1) ^ 1));   // nothing else to do: wait for the team
				if (stats_on) t_wait += clock64() - t0;
			}
			else break;
		}
		emit(PC_EXIT, 0, 0, nullptr, nullptr, false, false);
		flush();
		if (stats_on) {
			a.stats[blockIdx.x * 8 + 2] = t_wait;
			a.stats[blockIdx.x * 8 + 5] = clock64() - t_begin;
			a.stats[blockIdx.x * 8 + 6] = n_stages;
			a.stats[blockIdx.x * 8 + 7] = item_end - item0;
		}
	}
}

}  // namespace dspb200
