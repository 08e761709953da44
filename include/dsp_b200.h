/*
 * dsp_b200.h -- C ABI of libdspb200.so, the H100 (sm_90a) implementation of bmc0/dsp's
 * per-block effects-chain hot path.  Plain pointers and sizes only; no C++/torch types.
 *
 * What it replaces (reference file:line):
 *   run_effects_chain()/run_effect_list()           effects_chain.c:1044-1081
 *   biquad_effect_run[_all]() + biquad()            biquad.c:296-315, biquad.h:76-92
 *   fir_direct_effect_run(), fir_effect_run()       fir.c:43-62, fir.c:109-149
 *   fir_p_effect_run(), fft_part_group_compute()    fir_p.c:127-181, fir_p.c:64-103
 *   resample_effect_run(), resample_effect_drain2() resample.c:89-152, resample.c:163-188
 *   gain_effect_run()                               gain.c:25-33
 *   hilbert tap generator                           hilbert.c:65-77
 *
 * Data contract (same as the reference, dsp.h:42, effect.h:46): audio is IEEE double,
 * interleaved by frame: buf[frame * channels + channel].  All arithmetic on the device is
 * FP64.  State persists across calls (streaming); any frame count >= 1 per call is legal.
 *
 * A `dspb200_chain` is the device-side twin of one run of consecutive GPU effects of a
 * `struct effects_chain`: an ordered list of operators over `channels` interleaved channels.
 * Channels are independent for every operator here (EFFECT_FLAG_CH_DEPS_IDENTITY:
 * biquad.c:544, fir.c:237, fir_p.c:393, resample.c:264), so a chain is cut into contiguous
 * channel slabs ("shards"), each with its own full operator state on one GPU.  Host-buffer
 * calls do one strided scatter and one gather per shard (no collective, no NCCL).
 *
 * Error convention: functions returning int give 0 on success, negative on failure;
 * pointer-returning functions give NULL; frame-count functions give < 0 on failure (but see
 * dspb200_chain_drain_host).  dspb200_last_error() returns a thread-local message.  Nothing
 * here falls back to the CPU: without a usable CUDA device every constructor fails.
 */
#ifndef DSP_B200_H
#define DSP_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct dspb200_chain dspb200_chain;

/* ---- library / device ------------------------------------------------------------------ */
const char *dspb200_version(void);
const char *dspb200_last_error(void);
int  dspb200_device_count(void);                 /* CUDA devices visible; <= 0: none */
/* Pinned host memory for callers that want the fast host path (bench e2e, frontends). */
void *dspb200_host_alloc(size_t bytes);
void *dspb200_host_alloc_wc(size_t bytes);       /* write-combined variant for input-only buffers */
void  dspb200_host_free(void *p);
/* Number of kernels this library has launched so far in this process (all chains). */
long long dspb200_kernel_launches(void);

/* Per-kernel device timing for bench.py's roofline line: while enabled, the hot kernels are
 * bracketed by CUDA events on the stream they are launched on.  `name` is one of
 * "fir_mac", "fir_fwd", "fir_inv", "biquad", "resample", "edge" (the sample-format conversions); read() waits for the events, returns
 * the summed milliseconds and the launch count since the last read, and clears them. */
void dspb200_profile_enable(int on);
int  dspb200_profile_read(const char *name, double *total_ms, long *launches);
/* Measurement aid: while on, operators that normally overlap work on side streams enqueue everything on the
 * caller's stream, so per-kernel durations are free of contention (results are identical either way). */
void dspb200_debug_serialize(int on);
/* Test aid for the FIR's cross-stream ordering: while `roles` is non-zero, an FIR operator enqueues a delay of
 * `microseconds` (at most 5000) on each selected stream of its level-0 blocks blk % period == phase, right before that
 * stream's first FIR launch of the block, so that the stream falls behind the others.  Roles: the caller's stream (or
 * the shard's), the side stream (upper levels, per-block tail MAC), the second side stream (batch tiers) and the
 * look-ahead stream of the block kernel.  Results must not change.  roles = 0 turns it off (the default): then nothing
 * is added. */
enum { DSPB200_STALL_MAIN = 1, DSPB200_STALL_SIDE = 2, DSPB200_STALL_SIDE2 = 4, DSPB200_STALL_HOT = 8 };
int  dspb200_debug_stall(int roles, int microseconds, int period, int phase);

/* ---- chain construction ---------------------------------------------------------------- */
/* devices[n_devices]: CUDA ordinals to shard over (NULL/0: device 0).  slabs_per_device >= 1
 * cuts each device's channel range again so host-buffer calls overlap H2D, kernels and D2H. */
dspb200_chain *dspb200_chain_create(int fs, int channels, const int *devices, int n_devices,
                                    int slabs_per_device);
void dspb200_chain_destroy(dspb200_chain *c);
/* Move all operators of `src` to the end of `dest` (same fs/channels/sharding); `src` becomes
 * empty.  This is what an effect's merge() hook uses (effects_chain.c:605-641). */
int  dspb200_chain_absorb(dspb200_chain *dest, dspb200_chain *src);
int  dspb200_chain_n_ops(const dspb200_chain *c);
/* JSON description of the operators of shard 0 (plans, partition levels); returns its length. */
int  dspb200_chain_describe(const dspb200_chain *c, char *buf, size_t len);
int  dspb200_chain_n_shards(const dspb200_chain *c);
int  dspb200_chain_shard_info(const dspb200_chain *c, int shard, int *device, int *ch_begin, int *ch_count);
int  dspb200_chain_out_fs(const dspb200_chain *c);

/* gain.c:25-33 -- out = in * mult[ch] (+ add[ch] if add != NULL); unselected channels carry 1.0/0.0 */
int dspb200_chain_add_gain(dspb200_chain *c, const double *mult, const double *add);

/* biquad.c:296-315 -- cascade of n_stages TDF-II sections, coefs[stage][channel][5] =
 * {c0..c4} = {b0,b1,b2,a1,a2}/a0 (biquad.c:93-97).  A channel a stage does not act on carries
 * {1,0,0,0,0}.  The whole cascade is ONE pass over the block. */
int dspb200_chain_add_biquad(dspb200_chain *c, int n_stages, const double *coefs);

/* fir.c / fir_p.c -- out = in * taps (linear convolution, zero added latency), then delayed by
 * `latency` frames (fir.c's FFT path reports latency = len, fir.c:208-217; fir_p and the
 * direct form use 0).  selector[channels]: non-zero = filtered, zero = passed through
 * (NULL = all).  taps[filter_frames][filter_channels], filter_channels == 1 (shared) or ==
 * number of selected channels (column k -> k-th selected channel, fir.c:348-356).
 * block_hint: expected frames per call (0 = take it from the first call); the partition size
 * is the largest power of two <= hint within [64, 8192]. */
int dspb200_chain_add_fir(dspb200_chain *c, const char *selector, const double *taps,
                          int filter_channels, long filter_frames, long latency, long block_hint);

/* resample.c -- rational resampler fs -> out_fs with the reference's Albrecht-windowed sinc
 * (resample.c:52-87,274-316,361-366) evaluated as a polyphase FIR; bandwidth in [0.7,0.999]
 * (0 = default 0.939).  Emits exactly the frames resample_effect_run() would per call. */
int dspb200_chain_add_resample(dspb200_chain *c, int out_fs, double bandwidth);

/* align.c:35-64 / delay.c:47-63 -- channel k delayed by delay[k] >= 0 whole frames (0: untouched); the first
 * discard_frames frames of the stream are dropped (align.c:53-62, CLI build): such a call returns fewer frames. */
int dspb200_chain_add_align(dspb200_chain *c, const long *delay, long discard_frames);

/* 1 when every operator may run in place (dspb200_chain_run_host with in == out keeps the frame count). */
int dspb200_chain_inplace_ok(const dspb200_chain *c);

/* How many host->device / device->host block copies (one per shard and call) the library has issued so far. */
void dspb200_copy_counts(long long *h2d, long long *d2h);

/* ---- running --------------------------------------------------------------------------- */
/* Upper bound of output frames for `in_frames` input frames (effects_chain.c:993-1020). */
long dspb200_chain_max_out_frames(const dspb200_chain *c, long in_frames);

/* Mode A: host buffers, synchronous; in/out hold frames*channels (out: max_out_frames*channels)
 * doubles; in == out allowed.  Returns output frames. */
long dspb200_chain_run_host(dspb200_chain *c, long frames, const double *in, double *out);
/* The same work without the final wait (throughput frontends: file -> file, offline rendering).
 * Enqueues copy-in, the operators and copy-out of this block on the shards' streams and returns the
 * frame count `out` will hold; `in` and `out` must stay valid and untouched until
 * dspb200_chain_wait(chain, *ticket) (or dspb200_chain_sync) returns.  Blocks submitted back to back
 * overlap: copy-in of block k+1, kernels of block k and copy-out of block k-1 run concurrently
 * (use page-locked buffers, dspb200_host_alloc).  At most 8 tickets may be outstanding.
 * dspb200_chain_run_host == submit + wait; the two may be mixed freely. */
long dspb200_chain_submit_host(dspb200_chain *c, long frames, const double *in, double *out, unsigned long long *ticket);
int  dspb200_chain_wait(dspb200_chain *c, unsigned long long ticket);

/* Mode D: one shard, device-resident interleaved buffers of that shard's channel count,
 * enqueued on `stream` (a cudaStream_t; NULL = the legacy default stream), asynchronous.
 * d_in == d_out is allowed unless the chain's last operator changes the frame count (resample, align); such a call
 * is rejected before anything runs: it returns < 0 and leaves the buffer and the chain's state as they were.
 * Returns output frames.
 * Buffers: 8-byte alignment (that of a double) is enough for d_in and d_out; 16-byte-aligned rows may be faster.
 * d_in is never written unless the call is in place, and of d_out only the returned frames' rows are written.
 * Streams: every launch of the call waits for the work enqueued on `stream` before it, and `stream` waits for every
 * launch that reads d_in or writes d_out, so the caller may reuse both buffers in stream order as soon as the call
 * returns.  The results do not depend on the stream.  Calls of one chain made on different streams must be ordered by
 * the caller (an event recorded after one call, waited for before the next).  dspb200_chain_reset, _sync, _drain_host
 * and the host-buffer calls run on the library's own streams and are NOT ordered against Mode D work: synchronise
 * the device (or the streams of the Mode D calls) before making them. */
long dspb200_chain_run_device(dspb200_chain *c, int shard, long frames, const double *d_in,
                              double *d_out, void *stream);

/* Mode D timing aid: operators may keep look-ahead work on streams of their own (K2's tail MACs run one to
 * several block periods ahead of the block kernel).  Makes `stream` wait for everything shard `shard`'s operators
 * have enqueued so far, so that an event recorded on `stream` afterwards closes over ALL device work of the
 * calls made until now.  Not needed for correctness of later calls. */
int  dspb200_chain_join(dspb200_chain *c, int shard, void *stream);

/* Measurement hook: operator-specific device counters of operator `op_index` of shard `shard` (K2 with
 * DSP_B200_FIR_PIPE_STATS=1: per-CTA cycle counters of the last pipeline launch, 8 per CTA: team wait, MAC wait,
 * producer wait, team total, MAC total, producer total, stages, batch items).  Returns the count written. */
int  dspb200_debug_read(dspb200_chain *c, int shard, int op_index, long long *out, int max);

/* resample_effect_drain2() semantics (resample.c:163-188) for the whole chain: push zeros
 * until every rate-changing operator is dry.  Returns frames written (0..max_frames*ratio),
 * or -1 when nothing is left. */
long dspb200_chain_drain_host(dspb200_chain *c, long frames, double *out);

/* ---- sample formats at the edge -------------------------------------------------------- */
/* The _io variants of the four block calls take the caller's buffers in any of four formats, chosen independently
 * for input and output: a sample type | a layout.
 *   DSPB200_IO_F64 / DSPB200_IO_F32: IEEE double / float samples.
 *   interleaved (no layout bit): buf[frame * channels + channel], as everywhere else here; the stride is 0.
 *   DSPB200_IO_PLANAR: channel k's row starts at base + k * stride elements (numpy / torch [channels, frames]);
 *     stride >= frames on input, and >= dspb200_chain_max_out_frames(c, frames) on output.
 * Inside, every shard works on interleaved doubles as always; the conversion is one pass over the block on the
 * device (edge.cu), after the copy in and before the copy out.  It carries no policy: float -> double is exact,
 * double -> float rounds to nearest even with subnormals kept, values beyond FLT_MAX become +-Inf, and +-0, +-Inf
 * and NaN pass through (NaN payloads may be canonicalised).  f64 interleaved through an _io call is exactly the
 * plain call: no extra kernel, no staging copy.
 * Refusals: unknown format bits, a non-zero stride on an interleaved buffer, a short planar stride, and in == out with
 * a different format or stride on the two sides; each returns < 0 (-2 from drain_host_io) with a message in
 * dspb200_last_error() before anything is enqueued, and leaves the chain's state as it was.  Of the output only the
 * returned frames of each row are written; padding between planar rows is never touched.
 * Host calls: one host->device and one device->host copy per shard and call in every format (a planar shard's
 * channel slab is a run of consecutive rows: one 2-D copy); page-locking (DSP_B200_PIN) and the ticket ring work on
 * the caller's byte sizes.  Mode D: the buffers hold the shard's slab (a planar caller passes the address of the
 * slab's first row) and need only the alignment of their element type; the stream-ordering and "d_in is never
 * written unless in place" guarantees of dspb200_chain_run_device hold, as does its in-place rule. */
enum { DSPB200_IO_F64 = 0, DSPB200_IO_F32 = 1, DSPB200_IO_PLANAR = 0x10 };
long dspb200_chain_run_host_io(dspb200_chain *c, long frames, const void *in, int in_fmt, long in_stride,
                               void *out, int out_fmt, long out_stride);
long dspb200_chain_submit_host_io(dspb200_chain *c, long frames, const void *in, int in_fmt, long in_stride,
                                  void *out, int out_fmt, long out_stride, unsigned long long *ticket);
long dspb200_chain_run_device_io(dspb200_chain *c, int shard, long frames, const void *d_in, int in_fmt, long in_stride,
                                 void *d_out, int out_fmt, long out_stride, void *stream);
long dspb200_chain_drain_host_io(dspb200_chain *c, long frames, void *out, int out_fmt, long out_stride);

void dspb200_chain_reset(dspb200_chain *c);     /* effect->reset() of every operator */
int  dspb200_chain_sync(dspb200_chain *c);      /* wait for all shards' streams */

/* ---- init-time helpers that mirror reference host code ---------------------------------- */
/* Filter types and width types of biquad_init_using_type() (biquad.h:30-59; same numbering). */
enum {
	DSPB200_BQ_LOWPASS_1 = 1, DSPB200_BQ_HIGHPASS_1, DSPB200_BQ_ALLPASS_1, DSPB200_BQ_LOWSHELF_1,
	DSPB200_BQ_HIGHSHELF_1, DSPB200_BQ_LOWPASS_1P, DSPB200_BQ_LOWPASS, DSPB200_BQ_HIGHPASS,
	DSPB200_BQ_BANDPASS_SKIRT, DSPB200_BQ_BANDPASS_PEAK, DSPB200_BQ_NOTCH, DSPB200_BQ_ALLPASS,
	DSPB200_BQ_PEAK, DSPB200_BQ_LOWSHELF, DSPB200_BQ_HIGHSHELF, DSPB200_BQ_LOWPASS_TRANSFORM,
	DSPB200_BQ_HIGHPASS_TRANSFORM
};
enum {
	DSPB200_BQ_WIDTH_Q = 1, DSPB200_BQ_WIDTH_SLOPE, DSPB200_BQ_WIDTH_SLOPE_DB, DSPB200_BQ_WIDTH_BW_OCT,
	DSPB200_BQ_WIDTH_BW_HZ
};
/* biquad.c:91-294: c5 = {b0,b1,b2,a1,a2}/a0 for the given type (args as in the reference:
 * arg0 = f0 (or fz), arg1 = width (or qz), arg2 = gain dB (or fp), arg3 = qp). */
int dspb200_biquad_design(int type, double fs, double arg0, double arg1, double arg2, double arg3,
                          int width_type, double c5[5]);
/* hilbert.c:65-77: taps odd > 3; angle in radians (reference default -pi/2). */
int dspb200_hilbert_taps(long taps, double angle, double *h);
/* resample.c:274-316: derived parameters, for logs and tests.  out[8] =
 * {n, d, m, in_len, out_len, sinc_len, out_delay, taps_per_phase}. */
int dspb200_resample_params(int fs_in, int fs_out, double bandwidth, long out[8]);

/* ---- kernel unit-test hooks (used by tests/ only; device pointers) ----------------------- */
/* Packed real FFT of 2B points of B-sample blocks: in[n_ch][B] -> spec[n_ch][B] complex
 * (bin 0 packs DC.re, Nyquist.re), and back (first half + second half of the 2B result). */
int dspb200_test_rfft(int B, int n_ch, const double *d_in, double *d_spec, void *stream);
int dspb200_test_irfft(int B, int n_ch, const double *d_spec, double *d_out2B, void *stream);

#ifdef __cplusplus
}
#endif

#endif
