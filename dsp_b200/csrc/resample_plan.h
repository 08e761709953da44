// resample_plan.h -- K3: the resampler's parameters, the frame pacing of its calls and drain, and the launch each call gets:
// integer host code, tested without a device; resample.cu builds the tap table, keeps the input ring and launches.
#pragma once
#include <cmath>
#include <initializer_list>
#include <numeric>

namespace dspb200 {

struct ResampleParams { int n, d, m, in_len, out_len, sinc_len, out_delay, sinc_os, m_os; double fc_os; };

inline long next_smooth7(long n)
{
	for (;; ++n) {
		long m = n;
		for (int p : { 2, 3, 5, 7 })
			while (m % p == 0) m /= p;
		if (m == 1) return n;
	}
}

constexpr double ALBRECHT_M_FACT = 17.7822;
enum { RS_BAD_RATES = 1, RS_BAD_BANDWIDTH = 2 };

// resample.c:274-316; 0, or RS_BAD_RATES / RS_BAD_BANDWIDTH
inline int resample_params(int fs_in, int fs_out, double bw, ResampleParams *p)
{
	if (fs_in <= 0 || fs_out <= 0 || fs_in == fs_out) return RS_BAD_RATES;
	if (bw == 0.0) bw = 0.939;
	if (!(bw >= 0.7 && bw <= 0.999)) return RS_BAD_BANDWIDTH;
	const int max_rate = (fs_out > fs_in) ? fs_out : fs_in, min_rate = (fs_out > fs_in) ? fs_in : fs_out;
	const int g = std::gcd(fs_out, fs_in);
	p->n = fs_out / g, p->d = fs_in / g;
	const int max_factor = (p->n > p->d) ? p->n : p->d, min_factor = (p->n > p->d) ? p->d : p->n;
	p->m = (int) lround(2.0 * ALBRECHT_M_FACT * max_rate / (min_rate * (1.0 - bw)));
	const double width = ALBRECHT_M_FACT * max_rate / p->m;
	const double fc = (min_rate - width) / max_rate;
	p->sinc_os = (min_factor < 2) ? min_factor : 2;
	p->fc_os = fc / p->sinc_os;
	p->m_os = (p->m + 1) * p->sinc_os - 1;
	int len_mult = (p->m + 1) / max_factor + ((p->m + 1) % max_factor != 0);
	if (len_mult > 16) {
		const int fast = (int) next_smooth7(len_mult);
		if (fast != len_mult && (p->n <= 16 || p->d <= 16 || next_smooth7(p->n) == p->n || next_smooth7(p->d) == p->d))
			len_mult = fast;
	}
	p->sinc_len = max_factor * len_mult * p->sinc_os;
	p->in_len = p->d * len_mult;
	p->out_len = p->n * len_mult;
	p->out_delay = (fs_out == max_rate) ? p->m / 2 : (int) lround(p->m / 2 * ((double) p->n / p->d));
	return 0;
}

struct RsCall { long frames, first; };   // one call's emission: `frames` outputs from raw index `first` (< 0: stalled)

// resample.c:39-50's bookkeeping, in integers (the samples live in the operator's ring): the frames each call of
// resample_effect_run() emits (:91-151), reset() (:154-161) and drain2 (:163-188), so that every call emits exactly
// the frame count the reference would.
struct RsPacing {
	ResampleParams p{};
	long emit_pos = 0;          // next raw output index to emit
	int in_buf_pos = 0, out_buf_pos = 0, has_output = 0, is_draining = 0;
	long drain_pos = 0, drain_frames = 0;
	long max_out_frames(long in_frames) const { const long long r = (long long) in_frames * p.n; return (long) (r / p.d + (r % p.d != 0)); }

	RsCall run(long frames)
	{
		const long max_oframes = max_out_frames(frames);
		long iframes = 0, oframes = 0;
		while (iframes < frames) {
			long take = p.in_len - in_buf_pos;
			if (take > frames - iframes) take = frames - iframes;
			in_buf_pos += (int) take;
			iframes += take;
			if (has_output) {
				long emit = p.out_len - out_buf_pos;
				if (emit > max_oframes - oframes) emit = max_oframes - oframes;
				out_buf_pos += (int) emit;
				oframes += emit;
			}
			if (in_buf_pos == p.in_len && (!has_output || out_buf_pos == p.out_len)) {
				in_buf_pos = out_buf_pos = 0;
				if (!has_output) {
					out_buf_pos = p.out_delay;
					emit_pos += p.out_delay;   // only ever happens before the first emitted frame
					has_output = 1;
				}
			}
			else if (take == 0) return { -1, emit_pos };
		}
		emit_pos += oframes;
		return { oframes, emit_pos - oframes };   // emission is one contiguous raw range per call
	}
	// the drain counters are deliberately left alone, as in the reference
	void reset() { in_buf_pos = out_buf_pos = has_output = 0; emit_pos = 0; }
	// Before a drain poll: true when there is nothing (more) to flush.  The first poll fixes how many frames the drain
	// owes: the rest of the block being emitted, the delay line, and what the buffered input will make.
	bool drain_dry()
	{
		if (!has_output && in_buf_pos == 0) return true;
		if (!is_draining) {
			if (has_output) drain_frames += p.out_delay + p.out_len - out_buf_pos;
			drain_frames += max_out_frames(in_buf_pos);
			is_draining = 1;
		}
		return drain_pos >= drain_frames;
	}
	// After a poll that ran `produced` frames of silence: the part of them the drain still owes
	long drain_trim(long produced) { drain_pos += produced; return produced - ((drain_pos > drain_frames) ? drain_pos - drain_frames : 0); }
};

// ---- launch policy ----------------------------------------------------------------------------------------------
// DSP_B200_RS_TILE, read when the operator is made: 0 auto, 1..3 the FMA tiles (16x4, 16x2, 8x1), 4 tensor-core
// kernel, 5..7 the same with the tap tile double-buffered (cp.async) and the input rows requested 2 / 3 / 2 steps
// ahead at 4 / 3 / 3 CTAs per SM.  A forced tile the channel count cannot use falls back to the default.
constexpr int RS_DEFAULT_MMA = 7;   // 4: single-buffered tap tile; 7: double-buffered, input rows two steps ahead, 3 CTAs per SM (no spills)
constexpr int RS_MMA_Q = 32;        // output frames per CTA of the tensor-core kernels (RSM_Q)

// One launch of the resampler: the instantiation that runs, whose template arguments resample.cu reads from here
// (k_rs_poly<Q / warps, channels / 32, warps, minb> for tiles 1..3, k_rs_mma<warps> for 4, k_rs_mma2<warps, minb, depth>
// for 5..7), and its grid's tile, Q output frames by `channels` channels per CTA of 32 warps threads.  depth: input-row
// steps the tensor-core kernels request ahead of their use (0: FMA kernel); minb: CTAs per SM of the launch bounds.
struct RsLaunch { int tile = 0; const char *kernel = ""; int warps = 0, depth = 0, minb = 0, Q = 0, channels = 0; };

// the fixed shape of each variant; `warps` only matters to the tensor-core tiles
constexpr RsLaunch rs_variant(int tile, int warps)
{
	switch (tile) {
	case 1: return { 1, "k_rs_poly", 4, 0, 2, 64, 128 };   // 16 outputs x 4 channels per lane
	case 2: return { 2, "k_rs_poly", 2, 0, 6, 32, 64 };    // 16 x 2
	case 3: return { 3, "k_rs_poly", 4, 0, 4, 32, 32 };    // 8 x 1
	case 4: return { 4, "k_rs_mma", warps, 1, (warps == 4) ? 4 : 1, RS_MMA_Q, 32 * warps };
	default: return { tile, "k_rs_mma2", warps, (warps == 4 && tile == 6) ? 3 : 2, (warps < 4) ? 1 : (tile == 5) ? 4 : 3, RS_MMA_Q, 32 * warps };
	}
}

// The launch for a call that emits `oframes` frames on C channels, on a device of `sms` SMs
inline RsLaunch rs_launch(int C, long oframes, int sms, int force_tile)
{
	int tile = (C % 4 == 0) ? RS_DEFAULT_MMA : (C % 2 == 0) ? 2 : 3;
	if (force_tile >= 1 && force_tile <= 7 && !(((force_tile == 1 || force_tile >= 4) && C % 4) || (force_tile == 2 && C % 2))) tile = force_tile;
	// the tensor-core kernels: 4 warps (128 channels) per CTA as long as every SM still gets a few CTAs, else 2 or 1
	const long tiles = (oframes + RS_MMA_Q - 1) / RS_MMA_Q;
	const int warps = (C >= 128 && tiles * ((C + 127) / 128) >= 3L * sms) ? 4 : (C >= 64 && tiles * ((C + 63) / 64) >= 2L * sms) ? 2 : 1;
	return rs_variant(tile, warps);
}

}  // namespace dspb200
