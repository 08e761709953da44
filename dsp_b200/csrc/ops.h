// ops.h -- operator factories (one instance per shard); each lives in its own .cu file.
#pragma once
#include "common.cuh"

namespace dspb200 {

// gain.c:25-33
Op *make_gain_op(int slab_channels, int fs, const double *mult, const double *add);
// biquad.c:296-315; coefs[stage][slab_channels][5]
Op *make_biquad_op(int slab_channels, int fs, int n_stages, const double *coefs);
// returns a new operator equivalent to a followed by b, or nullptr if they cannot be fused (either has run
// since its last reset)
Op *fuse_biquad_ops(Op *a, Op *b);
// fir.c / fir_p.c; taps[filter_frames][filter_channels]; taps_cols[k] = filter column of the
// k-th selected channel of this slab (ignored when filter_channels == 1)
Op *make_fir_op(int slab_channels, int fs, const char *slab_selector, const double *taps, int filter_channels,
                long filter_frames, const int *taps_cols, long latency, long block_hint, cudaStream_t st);
// align.c:35-64 / delay.c:47-63: per-channel whole-sample delays (+ frames dropped at the head of the stream)
Op *make_align_op(int slab_channels, int fs, const long *delay, long discard_frames);
// resample.c
Op *make_resample_op(int slab_channels, int fs_in, int fs_out, double bandwidth, cudaStream_t st);

// resample_params() (resample_plan.h), which sets the library's error message when the rates or bandwidth are refused
struct ResampleParams;
int resample_params_or_error(int fs_in, int fs_out, double bw, ResampleParams *p);

// edge.cu: a block in the caller's format (io_plan.h; planar rows `stride` elements apart) <-> the working buffer, C
// channels of interleaved doubles; nothing is launched for f64 interleaved
void edge_in(int fmt, const void *src, long stride, double *dst, int C, long frames, cudaStream_t st);
void edge_out(int fmt, const double *src, void *dst, long stride, int C, long frames, cudaStream_t st);

void fir_debug_serialize(int on);
int fir_debug_stall(int roles, int us, int period, int phase);
int test_rfft(int B, int n_ch, const double *d_in, double *d_spec, cudaStream_t st);
int test_irfft(int B, int n_ch, const double *d_spec, double *d_out2B, cudaStream_t st);

}  // namespace dspb200
