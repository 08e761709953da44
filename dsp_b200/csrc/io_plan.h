// io_plan.h -- the sample-format edge's host decisions, tested without a device: which caller formats and strides a call
// accepts, each shard's host<->device copy geometry, the staging bytes a shard needs and which edge kernel
// (edge.cu) each side of a call runs.  api.cu takes every one of these from here.
//
// A format is a sample type | a layout (DSPB200_IO_* in include/dsp_b200.h):
//   interleaved: [frames][channels], the reference's own layout; the stride is 0.
//   planar:      channel k's row starts at base + k * stride elements, stride >= the frames the row holds.
// On the device a shard always works on interleaved doubles of its slab; f64 interleaved is that layout already and
// needs neither a kernel nor staging.  Every other format is copied raw (the caller's bytes, the shard's slab) into a
// staging buffer and converted there by the edge kernels.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstdio>

namespace dspb200 {

constexpr int IO_F64 = 0, IO_F32 = 1, IO_PLANAR = 0x10;
constexpr int IO_FMT_BITS = IO_F32 | IO_PLANAR;

inline bool io_fmt_ok(int fmt) { return (fmt & ~IO_FMT_BITS) == 0; }
inline size_t io_esize(int fmt) { return (fmt & IO_F32) ? 4 : 8; }
inline bool io_planar(int fmt) { return (fmt & IO_PLANAR) != 0; }

// The edge kernel a side runs: -1 for f64 interleaved (none), else the format itself (edge.cu's template over type and
// layout: IO_F32, IO_PLANAR (f64 planar) or IO_F32 | IO_PLANAR).
inline int io_kernel(int fmt) { return fmt == IO_F64 ? -1 : fmt; }

// Checks a call's formats and strides before anything is enqueued.  frames: the call's input frames; max_out: the
// chain's max_out_frames(frames); same_buffer: in == out.  Returns 0, or -1 with the reason in msg.
inline int io_check(int in_fmt, long in_stride, int out_fmt, long out_stride, long frames, long max_out, bool same_buffer,
                    char *msg, size_t len)
{
	if (!io_fmt_ok(in_fmt) || !io_fmt_ok(out_fmt)) {
		snprintf(msg, len, "io: unknown format bits (in 0x%x, out 0x%x; known: f32 0x1, planar 0x10)", (unsigned) in_fmt, (unsigned) out_fmt);
		return -1;
	}
	if (!io_planar(in_fmt) && in_stride != 0) {
		snprintf(msg, len, "io: interleaved input takes stride 0, got %ld", in_stride);
		return -1;
	}
	if (!io_planar(out_fmt) && out_stride != 0) {
		snprintf(msg, len, "io: interleaved output takes stride 0, got %ld", out_stride);
		return -1;
	}
	if (io_planar(in_fmt) && in_stride < frames) {
		snprintf(msg, len, "io: planar input stride %ld is shorter than the %ld frames of the call", in_stride, frames);
		return -1;
	}
	if (io_planar(out_fmt) && out_stride < max_out) {
		snprintf(msg, len, "io: planar output stride %ld is shorter than the chain's max_out_frames %ld", out_stride, max_out);
		return -1;
	}
	if (same_buffer && (in_fmt != out_fmt || in_stride != out_stride)) {
		snprintf(msg, len, "io: in place needs the same format and stride on both sides (in 0x%x/%ld, out 0x%x/%ld)",
		         (unsigned) in_fmt, in_stride, (unsigned) out_fmt, out_stride);
		return -1;
	}
	return 0;
}

// Mode D: a device buffer needs the alignment of its element type.
inline bool io_aligned(uintptr_t addr, int fmt) { return addr % io_esize(fmt) == 0; }

// One shard's copy of `frames` frames between the caller's host buffer of C channels and its device slab (byte units):
// `height` rows of `width` bytes, the host's rows `host_pitch` apart from host_off on, the device's `dev_pitch` apart.
// Interleaved: a row per frame, the shard's columns of it.  Planar: a row per channel of the slab, its first frames.
// The device side is always packed (a planar slab there has a pitch of `frames`).  contiguous: host and device rows
// both follow each other without a gap, one linear copy of width * height bytes does it.
struct IoCopy {
	size_t host_off = 0, host_pitch = 0, dev_pitch = 0, width = 0, height = 0;
	bool contiguous = false;
};

inline IoCopy io_copy(int fmt, long stride, int C, int ch_begin, int ch_count, long frames)
{
	const size_t e = io_esize(fmt);
	IoCopy k;
	if (io_planar(fmt)) {
		k.host_off = (size_t) ch_begin * stride * e;
		k.host_pitch = (size_t) stride * e;
		k.width = k.dev_pitch = (size_t) frames * e;
		k.height = (size_t) ch_count;
	}
	else {
		k.host_off = (size_t) ch_begin * e;
		k.host_pitch = (size_t) C * e;
		k.width = k.dev_pitch = (size_t) ch_count * e;
		k.height = (size_t) frames;
	}
	k.contiguous = k.host_pitch == k.width;
	return k;
}

// Bytes a host buffer of C channels in format `fmt` spans for rows of `frames` frames (what a call page-locks):
// interleaved frames * C elements, planar C - 1 whole strides and the last row's frames.
inline size_t io_host_bytes(int fmt, long stride, int C, long frames)
{
	const size_t n = io_planar(fmt) ? (size_t) (C - 1) * stride + frames : (size_t) frames * C;
	return n * io_esize(fmt);
}

// Staging bytes of a shard of ch_count channels for calls of `frames` input frames whose operators reach `max_frames`
// frames at most (Shard::walk_max_frames): the larger side, 0 when neither side converts.
inline size_t io_stage_bytes(int in_fmt, int out_fmt, int ch_count, long max_frames)
{
	const size_t in = io_kernel(in_fmt) < 0 ? 0 : (size_t) max_frames * ch_count * io_esize(in_fmt);
	const size_t out = io_kernel(out_fmt) < 0 ? 0 : (size_t) max_frames * ch_count * io_esize(out_fmt);
	return in > out ? in : out;
}

}  // namespace dspb200
