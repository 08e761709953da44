// edge.cu -- the sample-format edge: the caller's format (io_plan.h) <-> a shard's working buffer, interleaved doubles.
//
// k_edge_in converts the caller's block into the working buffer before the first operator, k_edge_out the last
// operator's result into the caller's format.  One template over (sample type, layout) covers f32 interleaved, f64
// planar and f32 planar; f64 interleaved is the working layout and runs neither.
//   interleaved f32: element-wise, 4 elements per thread; 128-bit loads and stores where both pointers allow them
//                    (a caller's f32 row may sit on any 4-byte boundary), coalesced scalar accesses otherwise.
//   planar:          a transpose through a 32 x 32 shared tile (rows padded to 33 doubles: the column reads of the
//                    64-bit tile are free of bank conflicts); each global read runs along a channel row or a frame,
//                    each write along the other; both ragged edges are bounds-checked.
// The conversions carry no policy: f32 -> f64 is exact, f64 -> f32 is __double2float_rn (round to nearest even,
// subnormals kept, beyond FLT_MAX -> +-Inf, the library is built without fast math); +-0, +-Inf and NaN pass.
#include "common.cuh"
#include "io_plan.h"
#include <cstdint>

namespace dspb200 {

constexpr int EDGE_TILE = 32, EDGE_ROWS = 8;   // planar: a 32 x 32 tile per CTA of 32 x 8 threads
constexpr int EDGE_THREADS = 256, EDGE_PER_THREAD = 4;

template <typename T> __device__ __forceinline__ double edge_to_f64(T v) { return (double) v; }
template <typename T> __device__ __forceinline__ T edge_from_f64(double v);
template <> __device__ __forceinline__ float edge_from_f64<float>(double v) { return __double2float_rn(v); }
template <> __device__ __forceinline__ double edge_from_f64<double>(double v) { return v; }

// 4 consecutive elements at p, 16-byte aligned
template <typename T> __device__ __forceinline__ void edge_load4(const T *p, double v[4])
{
	if constexpr (sizeof(T) == 4) {
		const float4 a = *reinterpret_cast<const float4 *>(p);
		v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
	}
	else {
		const double2 a = reinterpret_cast<const double2 *>(p)[0], b = reinterpret_cast<const double2 *>(p)[1];
		v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
	}
}

template <typename T> __device__ __forceinline__ void edge_store4(T *p, const double v[4])
{
	if constexpr (sizeof(T) == 4)
		*reinterpret_cast<float4 *>(p) = make_float4(__double2float_rn(v[0]), __double2float_rn(v[1]), __double2float_rn(v[2]), __double2float_rn(v[3]));
	else {
		reinterpret_cast<double2 *>(p)[0] = make_double2(v[0], v[1]);
		reinterpret_cast<double2 *>(p)[1] = make_double2(v[2], v[3]);
	}
}

// interleaved: dst[i] = src[i], i < total, converted; vec: both pointers allow 128-bit accesses of 4 elements
template <typename S, typename D>
__device__ __forceinline__ void edge_copy(const S *__restrict__ src, D *__restrict__ dst, long total, bool vec)
{
	const long base = (long) blockIdx.x * (EDGE_THREADS * EDGE_PER_THREAD);
	if (vec) {
		const long i = base + (long) threadIdx.x * EDGE_PER_THREAD;
		if (i + EDGE_PER_THREAD <= total) {
			double v[4];
			edge_load4(src + i, v);
			edge_store4(dst + i, v);
			return;
		}
		for (long k = i; k < total && k < i + EDGE_PER_THREAD; ++k) dst[k] = edge_from_f64<D>(edge_to_f64(src[k]));
		return;
	}
	for (int r = 0; r < EDGE_PER_THREAD; ++r) {
		const long k = base + r * EDGE_THREADS + threadIdx.x;
		if (k < total) dst[k] = edge_from_f64<D>(edge_to_f64(src[k]));
	}
}

// caller format -> working buffer [frames][C] doubles; planar rows `stride` elements apart
template <typename T, bool PLANAR>
__global__ void __launch_bounds__(EDGE_THREADS) k_edge_in(const T *__restrict__ src, long stride, double *__restrict__ dst, int C, long frames)
{
	if constexpr (!PLANAR) {
		const bool vec = ((uintptr_t) src % 16 == 0) && ((uintptr_t) dst % 16 == 0);
		edge_copy<T, double>(src, dst, frames * C, vec);
	}
	else {
		__shared__ double tile[EDGE_TILE][EDGE_TILE + 1];
		const long f0 = (long) blockIdx.x * EDGE_TILE;
		const int c0 = blockIdx.y * EDGE_TILE;
		for (int j = threadIdx.y; j < EDGE_TILE; j += EDGE_ROWS) {
			const int c = c0 + j;
			const long f = f0 + threadIdx.x;
			if (c < C && f < frames) tile[j][threadIdx.x] = edge_to_f64(src[(long) c * stride + f]);
		}
		__syncthreads();
		for (int j = threadIdx.y; j < EDGE_TILE; j += EDGE_ROWS) {
			const long f = f0 + j;
			const int c = c0 + threadIdx.x;
			if (c < C && f < frames) dst[f * C + c] = tile[threadIdx.x][j];
		}
	}
}

// working buffer [frames][C] doubles -> caller format; planar rows `stride` elements apart
template <typename T, bool PLANAR>
__global__ void __launch_bounds__(EDGE_THREADS) k_edge_out(const double *__restrict__ src, T *__restrict__ dst, long stride, int C, long frames)
{
	if constexpr (!PLANAR) {
		const bool vec = ((uintptr_t) src % 16 == 0) && ((uintptr_t) dst % 16 == 0);
		edge_copy<double, T>(src, dst, frames * C, vec);
	}
	else {
		__shared__ double tile[EDGE_TILE][EDGE_TILE + 1];
		const long f0 = (long) blockIdx.x * EDGE_TILE;
		const int c0 = blockIdx.y * EDGE_TILE;
		for (int j = threadIdx.y; j < EDGE_TILE; j += EDGE_ROWS) {
			const long f = f0 + j;
			const int c = c0 + threadIdx.x;
			if (c < C && f < frames) tile[j][threadIdx.x] = src[f * C + c];
		}
		__syncthreads();
		for (int j = threadIdx.y; j < EDGE_TILE; j += EDGE_ROWS) {
			const int c = c0 + j;
			const long f = f0 + threadIdx.x;
			if (c < C && f < frames) dst[(long) c * stride + f] = edge_from_f64<T>(tile[threadIdx.x][j]);
		}
	}
}

static dim3 edge_grid(int fmt, int C, long frames)
{
	if (io_planar(fmt)) return dim3((unsigned) ceil_div(frames, EDGE_TILE), (unsigned) ceil_div(C, EDGE_TILE));
	return dim3((unsigned) ceil_div(frames * C, EDGE_THREADS * EDGE_PER_THREAD));
}

static dim3 edge_block(int fmt) { return io_planar(fmt) ? dim3(EDGE_TILE, EDGE_ROWS) : dim3(EDGE_THREADS); }

void edge_in(int fmt, const void *src, long stride, double *dst, int C, long frames, cudaStream_t st)
{
	if (frames <= 0) return;
	ProfScope prof("edge", st);
	const dim3 g = edge_grid(fmt, C, frames), b = edge_block(fmt);
	switch (io_kernel(fmt)) {
	case IO_F32: LAUNCH((k_edge_in<float, false>), g, b, 0, st, (const float *) src, stride, dst, C, frames); break;
	case IO_PLANAR: LAUNCH((k_edge_in<double, true>), g, b, 0, st, (const double *) src, stride, dst, C, frames); break;
	case IO_F32 | IO_PLANAR: LAUNCH((k_edge_in<float, true>), g, b, 0, st, (const float *) src, stride, dst, C, frames); break;
	default: break;
	}
}

void edge_out(int fmt, const double *src, void *dst, long stride, int C, long frames, cudaStream_t st)
{
	if (frames <= 0) return;
	ProfScope prof("edge", st);
	const dim3 g = edge_grid(fmt, C, frames), b = edge_block(fmt);
	switch (io_kernel(fmt)) {
	case IO_F32: LAUNCH((k_edge_out<float, false>), g, b, 0, st, src, (float *) dst, stride, C, frames); break;
	case IO_PLANAR: LAUNCH((k_edge_out<double, true>), g, b, 0, st, src, (double *) dst, stride, C, frames); break;
	case IO_F32 | IO_PLANAR: LAUNCH((k_edge_out<float, true>), g, b, 0, st, src, (float *) dst, stride, C, frames); break;
	default: break;
	}
}

}  // namespace dspb200
