// fir_tile.cuh -- K2's device code shared by the FIR kernels (fir.cu) and the pipeline kernel (fir_pipe.cuh): the
// packed real-transform split and merge, the overlap-add, the MACs on packed rows, the sliding filter window, the
// FDL ring and the PTX primitives (mbarriers, bulk copies, cluster barriers).
//
// Spectra are stored "packed": N complex per row of a 2N-point real transform, bin 0 = (DC.re, Nyquist.re).  The
// transforms run as N-point complex FFTs in shared memory (fft.cuh) on z[n] = x[2n] + i x[2n+1]; the inverse is the
// same forward FFT of conj(Z), so the buffer holds conjugated values on the way in and out of it.
#pragma once
#include "fft.cuh"
#include <cstdint>

namespace dspb200 {

// ---- packed real transforms ------------------------------------------------------------------------------------

// Forward split of bin pair k out of the transform buffer: store(k, n, X[k], X[n]) with n = N - k; for k = 0 the
// packed bin 0 and n = N/2 (E = Re z, O = Im z, w = -i).  w = W_2N^k.
template <int N, class Store>
__device__ __forceinline__ void rfft_split(const double2 *buf, int k, double2 w, Store store)
{
	if (k == 0) {
		const double2 z0 = buf[0], zh = buf[spad(N / 2)];
		store(0, N / 2, make_double2(z0.x + z0.y, z0.x - z0.y), cconj(zh));
	}
	else {
		const double2 zk = buf[spad(k)], zn = buf[spad(N - k)];
		const double2 e = make_double2(0.5 * (zk.x + zn.x), 0.5 * (zk.y - zn.y));
		const double2 o = make_double2(0.5 * (zk.y + zn.y), -0.5 * (zk.x - zn.x));
		const double2 wo = cmul(w, o);
		store(k, N - k, cadd(e, wo), cconj(csub(e, wo)));
	}
}

// Inverse merge of bin pair k: S[k], S[n] (n = N - k, or N/2 for the packed bin 0) -> conj(Z[k]), conj(Z[n]) in the
// transform buffer, ready for the forward FFT.  w = W_2N^k.
template <int N>
__device__ __forceinline__ void irfft_merge(double2 *buf, int k, int n, const double2 &Sk, const double2 &Sn, const double2 &w)
{
	if (k == 0) {
		// Z[0] = E0 + i O0 from the packed (DC, Nyquist) pair; conj(Z[N/2]) = S[N/2]
		buf[0] = make_double2(0.5 * (Sk.x + Sk.y), -0.5 * (Sk.x - Sk.y));
		buf[spad(N / 2)] = Sn;
	}
	else {
		const double2 e = make_double2(0.5 * (Sk.x + Sn.x), 0.5 * (Sk.y - Sn.y));
		const double2 d = make_double2(0.5 * (Sk.x - Sn.x), 0.5 * (Sk.y + Sn.y));
		const double2 o = cmul(cconj(w), d);
		// Z[k] = E + iO, Z[N-k] = conj(E) + i conj(O); store conj(Z)
		buf[spad(k)] = make_double2(e.x - o.y, -(e.y + o.x));
		buf[spad(n)] = make_double2(e.x + o.y, -(o.x - e.y));
	}
}

// Overlap-add on the conjugated result of the inverse transform (scale = 1/N): the output pair of entry n of the first
// half plus the carry, and an entry of the second half scaled -- the next block's carry.
__device__ __forceinline__ double2 ola_out(double2 lo, double scale, double2 carry)
{
	return make_double2(fma(lo.x, scale, carry.x), fma(-lo.y, scale, carry.y));
}

__device__ __forceinline__ double2 ola_scaled(double2 hi, double scale) { return make_double2(hi.x * scale, -hi.y * scale); }

// ---- block I/O ---------------------------------------------------------------------------------------------------

// frames 2n, 2n+1 (n = t + i T) of one channel of an interleaved block, `stride` doubles between frames
template <int T>
__device__ __forceinline__ void read_frame_pairs(double2 (&v)[8], const double *xc, long stride, int t)
{
#pragma unroll
	for (int i = 0; i < 8; ++i) {
		const long n2 = 2L * (t + i * T);
		v[i] = make_double2(xc[n2 * stride], xc[(n2 + 1) * stride]);
	}
}

// a transform buffer from this thread's 8 frame pairs: the block in the first half, zeros in the second (v = NULL:
// the zeros only)
template <int N, int T>
__device__ __forceinline__ void fill_buf(double2 *buf, const double2 *v, int t)
{
#pragma unroll
	for (int i = 0; i < 8; ++i) {
		if (v) buf[spad(t + i * T)] = v[i];
		buf[spad(t + i * T + N / 2)] = make_double2(0.0, 0.0);
	}
}

// pull `bytes` starting at p towards L2, one request per 128-byte line, spread over T threads
__device__ __forceinline__ void prefetch_rows(const void *p, long bytes, int t, int T)
{
	const char *c = static_cast<const char *>(p);
	for (long off = (long) t * 128; off < bytes; off += (long) T * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(c + off));
}

// row of the FDL ring (`rows` rows) p blocks back from row `slot`, 0 <= p <= rows
__device__ __forceinline__ int ring_back(int slot, int p, int rows) { return (slot - p < 0) ? slot - p + rows : slot - p; }

// ---- MACs on packed rows ---------------------------------------------------------------------------------------

__device__ __forceinline__ double2 cmac(double2 acc, double2 x, double2 h)
{
	return make_double2(fma(x.x, h.x, fma(-x.y, h.y, acc.x)), fma(x.x, h.y, fma(x.y, h.x, acc.y)));
}

// acc += x . h; dc: x and h are the packed bin 0 (DC and Nyquist, both real): two real products instead of a complex one
__device__ __forceinline__ void cmac_packed(double2 &acc, double2 x, double2 h, bool dc)
{
	if (dc) {
		acc.x = fma(x.x, h.x, acc.x);
		acc.y = fma(x.y, h.y, acc.y);
	}
	else {
		acc.x = fma(x.x, h.x, fma(-x.y, h.y, acc.x));
		acc.y = fma(x.x, h.y, fma(x.y, h.x, acc.y));
	}
}

// One row x against a sliding window of filter rows: acc[t] += x . hw[t] for the entries whose bit t is set in `live`
// (entry t at acc[t * STRIDE], hw[t * STRIDE]: STRIDE > 1 walks column i of a [T][STRIDE] register array from
// &a[0][i], i.e. across its rows, which relies on the array's rows being contiguous).  A row meets only the filter rows of its window; the products with the
// other entries are skipped, not multiplied by zero -- an FDL row outside a period's window may hold a NaN or Inf (of
// a block that period does not depend on), and 0 x NaN would carry it into that period's sum.
template <int T, int STRIDE = 1>
__device__ __forceinline__ void window_mac(double2 *acc, const double2 *hw, unsigned live, const double2 &x, bool dc)
{
#pragma unroll
	for (int t = 0; t < T; ++t) {
		if (!((live >> t) & 1u)) continue;
		cmac_packed(acc[t * STRIDE], x, hw[t * STRIDE], dc);
	}
}

// ---- mbarrier / bulk-copy / cluster primitives (PTX; SASS: SYNCS.*, UBLKCP) ---------------------------------------

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, unsigned bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, unsigned parity)
{
	uint32_t ok;
	asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
	             : "=r"(ok)
	             : "r"(smem_u32(bar)), "r"(parity)
	             : "memory");
	return ok != 0;
}

// non-blocking probe (the MAC warps look at the NEXT stage before they work on the current one: its latency hides
// behind the arithmetic)
__device__ __forceinline__ bool mbar_test_wait(uint64_t *bar, unsigned parity)
{
	uint32_t ok;
	asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
	             : "=r"(ok)
	             : "r"(smem_u32(bar)), "r"(parity)
	             : "memory");
	return ok != 0;
}

// one lane of a converged warp (ptxas then knows the code under it is executed by a single thread: the bulk copies
// are issued straight from uniform registers instead of a per-lane loop)
__device__ __forceinline__ bool elect_one()
{
	uint32_t pred;
	asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
	return pred != 0;
}

// try_wait suspends the warp in hardware for a bounded time; a wait that has not come true after 2^20 of them (>= 50 ms) is a
// protocol bug: trap (the launch fails with an error) rather than hang the device
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity)
{
	unsigned spins = 0;
	while (!mbar_try_wait(bar, parity))
		if (++spins > (1u << 20)) __trap();
}

// wait for a phase completed by other CTAs' bulk copies (acquire at cluster scope); traps instead of hanging
__device__ __forceinline__ void mbar_wait_cluster(uint64_t *bar, unsigned parity)
{
	unsigned spins = 0;
	for (;;) {
		uint32_t ok;
		asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
		             : "=r"(ok)
		             : "r"(smem_u32(bar)), "r"(parity)
		             : "memory");
		if (ok) return;
		if (++spins > (1u << 20)) __trap();
	}
}

__device__ __forceinline__ uint64_t l2_policy_evict_first()
{
	uint64_t pol;
	asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
	return pol;
}

// global -> shared bulk copy, completion signalled on `bar` in bytes
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, uint64_t *bar, bool hint, uint64_t pol)
{
	if (hint)
		asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
		             "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
		             : "memory");
	else
		asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
		             "r"(bytes), "r"(smem_u32(bar))
		             : "memory");
}

__device__ __forceinline__ uint32_t mapa_u32(uint32_t cta_addr, uint32_t rank)
{
	uint32_t r;
	asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(cta_addr), "r"(rank));
	return r;
}

// `bytes` (a multiple of 16) from this CTA's shared memory into the shared memory of a CTA of the cluster; they count on
// that CTA's mbarrier when they have landed.  Issued by one thread.
__device__ __forceinline__ void bulk_s2c(uint32_t dst_cluster, uint32_t src_cta, unsigned bytes, uint32_t mbar_cluster)
{
	asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_cluster), "r"(src_cta),
	             "r"(bytes), "r"(mbar_cluster)
	             : "memory");
}

// generic-proxy writes to shared memory before, async-proxy (bulk copy) reads of them after
__device__ __forceinline__ void fence_proxy_async_smem()
{
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Cluster-wide execution barrier WITHOUT the release fence of cluster.sync(): for points where nothing written before
// has to become visible to the other CTAs (the fence of the releasing form waits for every global store and prefetch
// the thread still has in flight -- a third of the fused kernel's stall samples were that wait).
__device__ __forceinline__ void cluster_barrier_relaxed()
{
	asm volatile("barrier.cluster.arrive.relaxed.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
}

}  // namespace dspb200
