// api.cu -- the C ABI (include/dsp_b200.h): chains, shards, host/device run loops.
//
// A chain is the device-side twin of run_effect_list() (effects_chain.c:1044-1056): it walks
// its operators in order over one block, ping-ponging between buffers.  The difference is
// WHERE the block lives: it is copied to the GPU once, every operator of the chain works on it
// in HBM, and it is copied back once.  Channels are cut into shards (device x slab); each
// shard is an independent replica of the operator list over its channel slab with its own
// stream, so shards on one GPU overlap copies with kernels and shards on different GPUs run
// concurrently.  There is no cross-shard data dependency, hence no collective.
#include "common.cuh"
#include "ops.h"
#include "biquad_plan.h"
#include "resample_plan.h"
#include "io_plan.h"
#include "fft.cuh"
#include "../../include/dsp_b200.h"
#include <cassert>
#include <cmath>
#include <map>
#include <mutex>
#include <vector>

namespace dspb200 {

// ------------------------------------------------------------------------------------------
// errors, counters, twiddles
// ------------------------------------------------------------------------------------------
static thread_local char tls_error[512] = "";
std::atomic<long long> g_kernel_launches{0};

// ---- cache of freed device blocks (common.cuh: dev_alloc / dev_free) ----------------------------
namespace {
struct PoolState {
	std::mutex mu;
	std::map<void *, std::pair<int, size_t>> live;                 // block -> (device, bytes)
	std::multimap<std::pair<int, size_t>, void *> idle;            // (device, bytes) -> block
	size_t idle_bytes = 0;
	size_t cap = ((getenv("DSP_B200_POOL_MB") ? (size_t) atol(getenv("DSP_B200_POOL_MB")) : 8192)) << 20;
};
PoolState &pool()
{
	static PoolState *p = new PoolState();   // never destroyed: blocks may be freed from static destructors
	return *p;
}
}   // namespace

void *pool_alloc(size_t bytes)
{
	PoolState &ps = pool();
	int dev = 0;
	cudaGetDevice(&dev);
	{
		std::lock_guard<std::mutex> lk(ps.mu);
		auto it = ps.idle.find(std::make_pair(dev, bytes));
		if (it != ps.idle.end()) {
			void *p = it->second;
			ps.idle.erase(it);
			ps.idle_bytes -= bytes;
			ps.live[p] = std::make_pair(dev, bytes);
			return p;
		}
	}
	void *p = nullptr;
	cudaError_t err = cudaMalloc(&p, bytes);
	if (err != cudaSuccess) {
		// give the cache back to the driver and try once more
		std::vector<void *> drop;
		{
			std::lock_guard<std::mutex> lk(ps.mu);
			for (auto &kv : ps.idle) drop.push_back(kv.second);
			ps.idle.clear();
			ps.idle_bytes = 0;
		}
		cudaGetLastError();
		for (void *q : drop) cudaFree(q);
		err = cudaMalloc(&p, bytes);
	}
	if (err != cudaSuccess) {
		set_error("cudaMalloc(%zu bytes): %s", bytes, cudaGetErrorString(err));
		cudaGetLastError();
		return nullptr;
	}
	std::lock_guard<std::mutex> lk(ps.mu);
	ps.live[p] = std::make_pair(dev, bytes);
	return p;
}

void pool_free(void *p)
{
	PoolState &ps = pool();
	std::pair<int, size_t> info(0, 0);
	bool keep = false;
	{
		std::lock_guard<std::mutex> lk(ps.mu);
		auto it = ps.live.find(p);
		if (it != ps.live.end()) {
			info = it->second;
			ps.live.erase(it);
			keep = info.second >= (1u << 20) && ps.idle_bytes + info.second <= ps.cap;
		}
	}
	if (!keep) {
		cudaFree(p);
		return;
	}
	// cudaFree would have waited for the device: whatever still uses the block must be done before it is handed out again
	int cur = 0;
	cudaGetDevice(&cur);
	if (cur != info.first) cudaSetDevice(info.first);
	cudaDeviceSynchronize();
	if (cur != info.first) cudaSetDevice(cur);
	std::lock_guard<std::mutex> lk(ps.mu);
	ps.idle.insert(std::make_pair(info, p));
	ps.idle_bytes += info.second;
}
std::atomic<long long> g_h2d_copies{0}, g_d2h_copies{0};   // host<->device block copies issued (dspb200_copy_counts)

void set_error(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(tls_error, sizeof(tls_error), fmt, ap);
	va_end(ap);
	if (getenv("DSP_B200_VERBOSE")) fprintf(stderr, "dsp_b200: error: %s\n", tls_error);
}

const char *get_error() { return tls_error; }

static thread_local bool tls_launch_failed = false;

void note_launch_error(const char *kernel, cudaError_t err)
{
	set_error("launch of %s failed: %s", kernel, cudaGetErrorString(err));
	tls_launch_failed = true;
	cudaGetLastError();   // clear the non-sticky error so that later calls report their own
}

bool take_launch_error()
{
	const bool f = tls_launch_failed;
	tls_launch_failed = false;
	return f;
}

// per-kernel timing: pairs of events recorded around launches while profiling is enabled
std::atomic<int> g_profile_on{0};
namespace {
struct ProfRec { int device; cudaEvent_t a, b; bool closed; };
std::mutex g_prof_lock;
std::map<std::string, std::vector<ProfRec>> g_prof;
}

static std::vector<std::pair<cudaEvent_t, cudaEvent_t>> g_prof_pool;   // recycled event pairs (creation is slow)

void prof_mark(const char *name, cudaStream_t st, bool begin)
{
	std::lock_guard<std::mutex> lk(g_prof_lock);
	auto &v = g_prof[name];
	if (begin) {
		ProfRec r;
		r.closed = false;
		cudaGetDevice(&r.device);
		if (!g_prof_pool.empty()) {
			r.a = g_prof_pool.back().first;
			r.b = g_prof_pool.back().second;
			g_prof_pool.pop_back();
		}
		else if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess) return;
		cudaEventRecord(r.a, st);
		v.push_back(r);
	}
	else if (!v.empty() && !v.back().closed) {
		cudaEventRecord(v.back().b, st);
		v.back().closed = true;
	}
}

static std::mutex g_tw_lock;
static std::map<std::pair<int, int>, double2 *> g_tw;   // (device, N) -> table

const double2 *twiddles_2n(int N)
{
	int dev = 0;
	if (cudaGetDevice(&dev) != cudaSuccess) { set_error("no CUDA device"); return nullptr; }
	std::lock_guard<std::mutex> lk(g_tw_lock);
	auto it = g_tw.find({ dev, N });
	if (it != g_tw.end()) return it->second;
	std::vector<double2> h((size_t) 2 * N);
	for (int t = 0; t < 2 * N; ++t) {
		// exp(-2 pi i t / (2N)) with the argument reduced to [0, pi/4] for accuracy
		const long double a = 3.14159265358979323846264338327950288L * (long double) t / (long double) N;
		h[t].x = (double) cosl(a);
		h[t].y = (double) -sinl(a);
	}
	// exact values on the axes
	h[0] = make_double2(1.0, 0.0);
	h[N / 2] = make_double2(0.0, -1.0);
	h[N] = make_double2(-1.0, 0.0);
	h[3 * N / 2] = make_double2(0.0, 1.0);
	double2 *d = dev_alloc<double2>(h.size(), false);
	if (!d) return nullptr;
	CUDA_TRY(cudaMemcpy(d, h.data(), h.size() * sizeof(double2), cudaMemcpyHostToDevice), return nullptr);
	g_tw[{ dev, N }] = d;
	return d;
}

static std::map<std::pair<int, int>, double2 *> g_ptw;   // (device, N) -> per-pass tables

const double2 *twiddles_pass(int N)
{
	int dev = 0;
	if (cudaGetDevice(&dev) != cudaSuccess) { set_error("no CUDA device"); return nullptr; }
	std::lock_guard<std::mutex> lk(g_tw_lock);
	auto it = g_ptw.find({ dev, N });
	if (it != g_ptw.end()) return it->second;
	std::vector<double2> h((size_t) fft_pass_table_size(N) + 1);
	const long double pi = 3.14159265358979323846264338327950288L;
	size_t off = 0;
	long ns = 1;
	for (int p = 0; p < 4 && fft_radix(N, p) != 0; ++p) {
		const int R = fft_radix(N, p);
		if (ns > 1) {
			for (int mi = 0; mi < 4; ++mi)
				for (long k = 0; k < ns; ++k) {
					// exp(-2 pi i k 2^mi / (ns R)), argument reduced modulo one turn first
					const long num = (k << mi) % (ns * R);
					const long double ang = 2.0L * pi * (long double) num / (long double) (ns * R);
					h[off + (size_t) mi * ns + k] = make_double2((double) cosl(ang), (double) -sinl(ang));
				}
			off += 4 * ns;
		}
		ns *= R;
	}
	double2 *d = dev_alloc<double2>(h.size(), false);
	if (!d) return nullptr;
	CUDA_TRY(cudaMemcpy(d, h.data(), h.size() * sizeof(double2), cudaMemcpyHostToDevice), return nullptr);
	g_ptw[{ dev, N }] = d;
	return d;
}

// ------------------------------------------------------------------------------------------
// K4: gain.c:25-33
// ------------------------------------------------------------------------------------------
__global__ void k_gain(const double *in, double *out, const double *mult, const double *add, int C, long total)
{
	const long i = (long) blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= total) return;
	const int c = (int) (i % C);
	out[i] = fma(in[i], mult[c], add[c]);
}

struct GainOp : Op {
	double *d_mult = nullptr, *d_add = nullptr;
	const char *name() const override { return "gain"; }
	~GainOp() override { dev_free(d_mult); dev_free(d_add); }
	void reset(cudaStream_t) override {}
	long run(long frames, const double *in, double *out, cudaStream_t st) override
	{
		const long total = frames * channels;
		if (total > 0) LAUNCH(k_gain, ceil_div(total, 256), 256, 0, st, in, out, d_mult, d_add, channels, total);
		return frames;
	}
};

Op *make_gain_op(int slab_channels, int fs, const double *mult, const double *add)
{
	std::unique_ptr<GainOp> op(new GainOp());
	op->channels = slab_channels;
	op->fs_in = op->fs_out = fs;
	op->d_mult = dev_alloc<double>(slab_channels, false);
	op->d_add = dev_alloc<double>(slab_channels, true);
	if (!op->d_mult || !op->d_add) return nullptr;
	CUDA_TRY(cudaMemcpy(op->d_mult, mult, slab_channels * sizeof(double), cudaMemcpyHostToDevice), return nullptr);
	if (add) CUDA_TRY(cudaMemcpy(op->d_add, add, slab_channels * sizeof(double), cudaMemcpyHostToDevice), return nullptr);
	return op.release();
}

// ------------------------------------------------------------------------------------------
// chain
// ------------------------------------------------------------------------------------------
struct Shard {
	int device = 0, ch_begin = 0, ch_count = 0;
	cudaStream_t stream = nullptr;
	std::vector<std::unique_ptr<Op>> ops;
	double *buf[4] = { nullptr, nullptr, nullptr, nullptr };   // io-in, io-out/scratch, scratch, zeros
	size_t cap = 0;   // doubles per buffer
	void *stage = nullptr;   // host calls in another format than f64 interleaved: the caller's raw slab (io_plan.h)
	size_t stage_cap = 0;    // bytes
	static constexpr int DONE_RING = 8;
	cudaEvent_t done[DONE_RING] = {};   // completion markers of submitted host blocks (ticket % DONE_RING)

	~Shard()
	{
		cudaSetDevice(device);
		ops.clear();
		for (double *b : buf) dev_free(b);
		dev_free(stage);
		for (cudaEvent_t e : done) if (e) cudaEventDestroy(e);
		if (stream) cudaStreamDestroy(stream);
	}

	long walk_max_frames(long frames, long *out_frames) const
	{
		long f = frames, mx = frames;
		for (const auto &op : ops) {
			f = op->max_out_frames(f);
			if (f > mx) mx = f;
		}
		if (out_frames) *out_frames = f;
		return mx;
	}

	// the working buffers for calls of `frames` frames, and the staging buffer of a host call in formats in_fmt / out_fmt
	int ensure_cap(long frames, int in_fmt = IO_F64, int out_fmt = IO_F64)
	{
		const long mx = walk_max_frames(frames, nullptr);
		const size_t need = (size_t) mx * ch_count, stage_need = io_stage_bytes(in_fmt, out_fmt, ch_count, mx);
		if (need <= cap && stage_need <= stage_cap) return 0;
		CUDA_TRY(cudaStreamSynchronize(stream), return -1);
		if (need > cap) {
			for (double *&b : buf) {
				dev_free(b);
				b = dev_alloc<double>(need, false);
				if (!b) { cap = 0; return -1; }
			}
			cap = need;
		}
		if (stage_need > stage_cap) {
			dev_free(stage);
			stage = dev_alloc<char>(stage_need, false);
			if (!stage) { stage_cap = 0; return -1; }
			stage_cap = stage_need;
		}
		return 0;
	}

	// run ops[first..) over `frames` frames: in -> out (device pointers, this shard's slab)
	long run_ops(size_t first, long frames, const double *in, double *out, bool in_writable, cudaStream_t st, bool host_mode = true)
	{
		for (auto &op : ops) op->host_mode = host_mode;
		const double *cur = in;
		bool cur_writable = in_writable || (in == out);
		long f = frames;
		int flip = 0;
		if (first >= ops.size()) {
			if (in != out && f > 0)
				CUDA_TRY(cudaMemcpyAsync(out, in, (size_t) f * ch_count * sizeof(double), cudaMemcpyDeviceToDevice, st), return -1);
			return f;
		}
		for (size_t i = first; i < ops.size(); ++i) {
			Op *op = ops[i].get();
			const bool last = (i + 1 == ops.size());
			double *dst;
			if (op->inplace_ok) {
				if (last) dst = out;
				else if (cur_writable) dst = const_cast<double *>(cur);
				else { dst = buf[1 + flip]; flip ^= 1; }
			}
			else {
				if (last) {
					// never in place: dspb200_chain_run_device rejects in == out on such a chain before anything runs,
					// and the host calls write their result to buf[3], which no operator reads
					assert(cur != out);
					dst = out;
				}
				else {
					dst = buf[1 + flip];
					flip ^= 1;
					if (dst == cur) { dst = buf[1 + flip]; flip ^= 1; }
				}
			}
			if (f > 0) {
				f = op->run(f, cur, dst, st);
				if (take_launch_error()) return -1;   // message already set by LAUNCH
				if (f < 0) return -1;
			}
			cur = dst;
			cur_writable = true;
		}
		return f;
	}
};

}  // namespace dspb200

using namespace dspb200;

static_assert(DSPB200_IO_F64 == IO_F64 && DSPB200_IO_F32 == IO_F32 && DSPB200_IO_PLANAR == IO_PLANAR, "io_plan.h follows the ABI");

struct dspb200_chain {
	int fs = 0, channels = 0;
	int out_fs = 0;
	int n_ops = 0;
	std::vector<std::unique_ptr<Shard>> shards;
	std::vector<std::pair<void *, size_t>> registered;    // host ranges pinned by us
	bool pin_host = false;
	unsigned long long ticket = 0;   // blocks submitted so far (dspb200_chain_submit_host); bumped only by a complete submission
	unsigned long long waited = 0;   // highest ticket known to be complete

	~dspb200_chain()
	{
		shards.clear();
		for (auto &r : registered) cudaHostUnregister(r.first);
	}
};

// The operators run work on several streams at once (K2: block kernel, look-ahead MAC, batched MAC).  CUDA multiplexes
// streams onto a small number of hardware queues (8 by default); in a process that has created and destroyed many
// streams, two streams of one operator can land on the same queue and silently serialise.  Ask for more queues
// before the CUDA context exists (no effect if the host application already decided, or initialised CUDA first).
__attribute__((constructor)) static void dspb200_more_hw_queues()
{
	setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
}

static bool g_probe_ok()
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) {
		set_error("no usable CUDA device (this library has no CPU path)");
		cudaGetLastError();
		return false;
	}
	return true;
}

extern "C" {

const char *dspb200_version(void) { return "dsp_b200 0.1 (sm_90a)"; }
const char *dspb200_last_error(void) { return get_error(); }

int dspb200_device_count(void)
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
	return n;
}

void *dspb200_host_alloc(size_t bytes)
{
	void *p = nullptr;
	if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) {
		set_error("cudaHostAlloc(%zu) failed", bytes);
		cudaGetLastError();
		return nullptr;
	}
	return p;
}

void *dspb200_host_alloc_wc(size_t bytes)
{
	// write-combined: faster for the GPU to read over PCIe, slow for the CPU to read back -- input buffers only
	void *p = nullptr;
	if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable | cudaHostAllocWriteCombined) != cudaSuccess) {
		set_error("cudaHostAlloc(%zu, write-combined) failed", bytes);
		cudaGetLastError();
		return nullptr;
	}
	return p;
}

void dspb200_host_free(void *p)
{
	if (p) cudaFreeHost(p);
}

long long dspb200_kernel_launches(void) { return g_kernel_launches.load(); }

void dspb200_profile_enable(int on) { g_profile_on.store(on ? 1 : 0); }

void dspb200_debug_serialize(int on) { fir_debug_serialize(on); }

int dspb200_debug_stall(int roles, int microseconds, int period, int phase) { return fir_debug_stall(roles, microseconds, period, phase); }

int dspb200_profile_read(const char *name, double *total_ms, long *launches)
{
	std::lock_guard<std::mutex> lk(g_prof_lock);
	double ms = 0.0;
	long n = 0;
	auto it = g_prof.find(name ? name : "");
	if (it != g_prof.end()) {
		for (auto &r : it->second) {
			if (r.closed) {
				cudaSetDevice(r.device);
				float t = 0.0f;
				if (cudaEventSynchronize(r.b) == cudaSuccess && cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) { ms += t; ++n; }
			}
			g_prof_pool.push_back({ r.a, r.b });   // single-device use: events go back to the pool
		}
		it->second.clear();
	}
	if (total_ms) *total_ms = ms;
	if (launches) *launches = n;
	return 0;
}

dspb200_chain *dspb200_chain_create(int fs, int channels, const int *devices, int n_devices, int slabs_per_device)
{
	if (!g_probe_ok()) return nullptr;
	if (channels < 1 || fs < 1) { set_error("chain: bad stream %d Hz x %d ch", fs, channels); return nullptr; }
	const int dev0 = 0;
	if (!devices || n_devices < 1) { devices = &dev0; n_devices = 1; }
	if (slabs_per_device < 1) slabs_per_device = 1;
	int n_shards = n_devices * slabs_per_device;
	if (n_shards > channels) n_shards = channels;
	std::unique_ptr<dspb200_chain> c(new dspb200_chain());
	c->fs = c->out_fs = fs;
	c->channels = channels;
	// Page-locking the CALLER's buffers is opt-in (DSP_B200_PIN=1; the C shim turns it on for the
	// frontends' long-lived block buffers): a stale registration over recycled heap memory makes
	// later copies fail, so arbitrary callers get plain pageable copies.
	const char *pin = getenv("DSP_B200_PIN");
	c->pin_host = (pin && pin[0] == '1');
	for (int i = 0; i < n_shards; ++i) {
		std::unique_ptr<Shard> s(new Shard());
		s->device = devices[(long) i * n_devices / n_shards];
		s->ch_begin = (int) ((long) channels * i / n_shards);
		s->ch_count = (int) ((long) channels * (i + 1) / n_shards) - s->ch_begin;
		CUDA_TRY(cudaSetDevice(s->device), return nullptr);
		CUDA_TRY(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking), return nullptr);
		c->shards.push_back(std::move(s));
	}
	return c.release();
}

void dspb200_chain_destroy(dspb200_chain *c) { delete c; }

int dspb200_chain_absorb(dspb200_chain *dest, dspb200_chain *src)
{
	if (!dest || !src || dest == src) return -1;
	if (dest->out_fs != src->fs || dest->channels != src->channels || dest->shards.size() != src->shards.size()) {
		set_error("chain_absorb: incompatible chains");
		return -1;
	}
	for (size_t i = 0; i < dest->shards.size(); ++i) {
		Shard &a = *dest->shards[i], &b = *src->shards[i];
		if (a.device != b.device || a.ch_begin != b.ch_begin || a.ch_count != b.ch_count) {
			set_error("chain_absorb: shard layout differs");
			return -1;
		}
	}
	for (size_t i = 0; i < dest->shards.size(); ++i) {
		Shard &a = *dest->shards[i], &b = *src->shards[i];
		cudaSetDevice(b.device);
		cudaStreamSynchronize(b.stream);
		for (auto &op : b.ops) {
			// cascaded biquads collapse into one fused operator (biquad.cu); everything else queues up
			Op *fused = a.ops.empty() ? nullptr : fuse_biquad_ops(a.ops.back().get(), op.get());
			if (fused) a.ops.back().reset(fused);
			else a.ops.push_back(std::move(op));
		}
		b.ops.clear();
	}
	dest->n_ops = (int) dest->shards[0]->ops.size();
	dest->out_fs = src->out_fs;
	src->n_ops = 0;
	src->out_fs = src->fs;
	return 0;
}

int dspb200_chain_describe(const dspb200_chain *c, char *buf, size_t len)
{
	if (!c || !buf || len == 0) return -1;
	std::string s = "[";
	if (!c->shards.empty()) {
		bool first = true;
		for (const auto &op : c->shards[0]->ops) {
			if (!first) s += ",";
			s += op->describe();
			first = false;
		}
	}
	s += "]";
	snprintf(buf, len, "%s", s.c_str());
	return (int) s.size();
}

int dspb200_chain_n_ops(const dspb200_chain *c) { return c ? c->n_ops : 0; }
int dspb200_chain_n_shards(const dspb200_chain *c) { return c ? (int) c->shards.size() : 0; }
int dspb200_chain_out_fs(const dspb200_chain *c) { return c ? c->out_fs : 0; }

int dspb200_chain_shard_info(const dspb200_chain *c, int shard, int *device, int *ch_begin, int *ch_count)
{
	if (!c || shard < 0 || shard >= (int) c->shards.size()) return -1;
	const Shard &s = *c->shards[shard];
	if (device) *device = s.device;
	if (ch_begin) *ch_begin = s.ch_begin;
	if (ch_count) *ch_count = s.ch_count;
	return 0;
}

#define FOR_EACH_SHARD(c, s) for (auto &s##_p : (c)->shards) if (Shard *s = s##_p.get())

int dspb200_chain_add_gain(dspb200_chain *c, const double *mult, const double *add)
{
	if (!c || !mult) return -1;
	FOR_EACH_SHARD(c, s) {
		CUDA_TRY(cudaSetDevice(s->device), return -1);
		Op *op = make_gain_op(s->ch_count, c->out_fs, mult + s->ch_begin, add ? add + s->ch_begin : nullptr);
		if (!op) return -1;
		s->ops.emplace_back(op);
	}
	++c->n_ops;
	return 0;
}

int dspb200_chain_add_biquad(dspb200_chain *c, int n_stages, const double *coefs)
{
	if (!c || !coefs || n_stages < 1) return -1;
	const int C = c->channels;
	// long cascades are cut into operators of <= BQ_MAX_STAGES stages
	for (int st0 = 0; st0 < n_stages; st0 += BQ_MAX_STAGES) {
		const int ns = (n_stages - st0 < BQ_MAX_STAGES) ? n_stages - st0 : BQ_MAX_STAGES;
		FOR_EACH_SHARD(c, s) {
			CUDA_TRY(cudaSetDevice(s->device), return -1);
			std::vector<double> slab((size_t) ns * s->ch_count * 5);
			for (int st = 0; st < ns; ++st)
				memcpy(&slab[(size_t) st * s->ch_count * 5], &coefs[((size_t) (st0 + st) * C + s->ch_begin) * 5], (size_t) s->ch_count * 5 * sizeof(double));
			Op *op = make_biquad_op(s->ch_count, c->out_fs, ns, slab.data());
			if (!op) return -1;
			s->ops.emplace_back(op);
		}
		++c->n_ops;
	}
	return 0;
}

int dspb200_chain_add_fir(dspb200_chain *c, const char *selector, const double *taps, int filter_channels,
                          long filter_frames, long latency, long block_hint)
{
	if (!c || !taps || filter_frames < 1 || filter_channels < 1 || latency < 0) { set_error("fir: bad arguments"); return -1; }
	const int C = c->channels;
	int n_sel = 0;
	for (int k = 0; k < C; ++k) n_sel += (!selector || selector[k]) ? 1 : 0;
	if (filter_channels != 1 && filter_channels != n_sel) {
		// fir.c:221-225
		set_error("fir: channels mismatch: channels=%d filter_channels=%d", n_sel, filter_channels);
		return -1;
	}
	int sel_before = 0;
	FOR_EACH_SHARD(c, s) {
		CUDA_TRY(cudaSetDevice(s->device), return -1);
		std::vector<int> cols;
		for (int k = 0; k < s->ch_count; ++k)
			if (!selector || selector[s->ch_begin + k]) cols.push_back(sel_before++);
		Op *op = make_fir_op(s->ch_count, c->out_fs, selector ? selector + s->ch_begin : nullptr, taps, filter_channels,
		                     filter_frames, cols.data(), latency, block_hint, s->stream);
		if (!op) return -1;
		s->ops.emplace_back(op);
	}
	++c->n_ops;
	return 0;
}

int dspb200_chain_add_align(dspb200_chain *c, const long *delay, long discard_frames)
{
	if (!c || !delay || discard_frames < 0) { set_error("align: bad arguments"); return -1; }
	FOR_EACH_SHARD(c, s) {
		CUDA_TRY(cudaSetDevice(s->device), return -1);
		Op *op = make_align_op(s->ch_count, c->out_fs, delay + s->ch_begin, discard_frames);
		if (!op) return -1;
		s->ops.emplace_back(op);
	}
	++c->n_ops;
	return 0;
}

int dspb200_chain_inplace_ok(const dspb200_chain *c)
{
	if (!c || c->shards.empty()) return 1;
	for (const auto &op : c->shards[0]->ops)
		if (!op->inplace_ok) return 0;
	return 1;
}

void dspb200_copy_counts(long long *h2d, long long *d2h)
{
	if (h2d) *h2d = g_h2d_copies.load();
	if (d2h) *d2h = g_d2h_copies.load();
}

int dspb200_chain_add_resample(dspb200_chain *c, int out_fs, double bandwidth)
{
	if (!c) return -1;
	if (out_fs == c->out_fs) return 0;   // resample.c:256-259: same rate, effect dropped
	FOR_EACH_SHARD(c, s) {
		CUDA_TRY(cudaSetDevice(s->device), return -1);
		Op *op = make_resample_op(s->ch_count, c->out_fs, out_fs, bandwidth, s->stream);
		if (!op) return -1;
		s->ops.emplace_back(op);
	}
	c->out_fs = out_fs;
	++c->n_ops;
	return 0;
}

long dspb200_chain_max_out_frames(const dspb200_chain *c, long in_frames)
{
	if (!c || c->shards.empty()) return in_frames;
	long out = in_frames;
	c->shards[0]->walk_max_frames(in_frames, &out);
	return out;
}

static void maybe_pin(dspb200_chain *c, const void *p, size_t bytes)
{
	// The frontends' block buffers are plain calloc() memory that stays put between REALLOCs
	// (dsp.c:1067-1081, ladspa_dsp.c:322-338): page-lock them once so the copies are true DMA.
	if (!c->pin_host || !p || bytes == 0) return;
	for (auto &r : c->registered) {
		if (r.first != p) continue;
		if (r.second >= bytes) return;
		cudaHostUnregister(r.first);
		if (cudaHostRegister(r.first, bytes, cudaHostRegisterPortable) == cudaSuccess) r.second = bytes;
		else { cudaGetLastError(); r.second = 0; }
		return;
	}
	cudaPointerAttributes attr;
	if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { cudaGetLastError(); return; }
	if (attr.type != cudaMemoryTypeUnregistered) return;
	if (cudaHostRegister(const_cast<void *>(p), bytes, cudaHostRegisterPortable) == cudaSuccess)
		c->registered.push_back({ const_cast<void *>(p), bytes });
	else cudaGetLastError();
}

// One H2D (host_in) or D2H (host_out) copy of `frames` frames of a shard's slab between the caller's buffer in format
// `fmt` (planar rows `stride` elements apart) and the packed device slab `dev` (io_plan.h: io_copy).
static int copy_slab(const Shard &s, int C, int fmt, long stride, long frames, void *dev, const void *host_in, void *host_out)
{
	if (frames <= 0) return 0;
	const IoCopy k = io_copy(fmt, stride, C, s.ch_begin, s.ch_count, frames);
	(host_in ? g_h2d_copies : g_d2h_copies).fetch_add(1, std::memory_order_relaxed);
	if (host_in) {
		const char *h = static_cast<const char *>(host_in) + k.host_off;
		if (k.contiguous) CUDA_TRY(cudaMemcpyAsync(dev, h, k.width * k.height, cudaMemcpyHostToDevice, s.stream), return -1);
		else CUDA_TRY(cudaMemcpy2DAsync(dev, k.dev_pitch, h, k.host_pitch, k.width, k.height, cudaMemcpyHostToDevice, s.stream), return -1);
	}
	else {
		char *h = static_cast<char *>(host_out) + k.host_off;
		if (k.contiguous) CUDA_TRY(cudaMemcpyAsync(h, dev, k.width * k.height, cudaMemcpyDeviceToHost, s.stream), return -1);
		else CUDA_TRY(cudaMemcpy2DAsync(h, k.host_pitch, dev, k.dev_pitch, k.width, k.height, cudaMemcpyDeviceToHost, s.stream), return -1);
	}
	return 0;
}

static bool io_refused(int in_fmt, long in_stride, int out_fmt, long out_stride, long frames, long max_out, bool same_buffer)
{
	char msg[256];
	if (!io_check(in_fmt, in_stride, out_fmt, out_stride, frames, max_out, same_buffer, msg, sizeof(msg))) return false;
	set_error("%s", msg);
	return true;
}

long dspb200_chain_submit_host_io(dspb200_chain *c, long frames, const void *in, int in_fmt, long in_stride, void *out, int out_fmt,
                                  long out_stride, unsigned long long *ticket)
{
	if (!c || !in || !out) return -1;
	if (frames < 1) return 0;
	const int C = c->channels;
	const long max_out = dspb200_chain_max_out_frames(c, frames);
	if (io_refused(in_fmt, in_stride, out_fmt, out_stride, frames, max_out, in == out)) return -1;
	maybe_pin(c, in, io_host_bytes(in_fmt, in_stride, C, frames));
	if (out != in) maybe_pin(c, out, io_host_bytes(out_fmt, out_stride, C, io_planar(out_fmt) ? max_out : (max_out > frames) ? max_out : frames));
	const bool conv_in = io_kernel(in_fmt) >= 0, conv_out = io_kernel(out_fmt) >= 0;
	long result = -1;
	const unsigned long long t = c->ticket + 1;   // becomes current only when every shard has been enqueued
	if (ticket && t > c->waited + Shard::DONE_RING) {
		// the completion markers are a ring of DONE_RING: the oldest outstanding block is waited for here
		// rather than letting its marker be overwritten
		if (dspb200_chain_wait(c, t - Shard::DONE_RING)) return -1;
	}
	FOR_EACH_SHARD(c, s) {
		CUDA_TRY(cudaSetDevice(s->device), return -1);
		if (s->ensure_cap(frames, in_fmt, out_fmt)) return -1;
		// the staging buffer holds the caller's raw slab (a planar one with rows of `frames`, then `f` frames)
		if (copy_slab(*s, C, in_fmt, in_stride, frames, conv_in ? s->stage : s->buf[0], in, nullptr)) return -1;
		if (conv_in) {
			edge_in(in_fmt, s->stage, frames, s->buf[0], s->ch_count, frames, s->stream);
			if (take_launch_error()) return -1;
		}
		bool rate_change = false;
		for (auto &op : s->ops) rate_change |= !op->inplace_ok;
		double *dst = rate_change ? s->buf[3] : s->buf[0];
		const long f = s->run_ops(0, frames, s->buf[0], dst, true, s->stream, /* one block at a time: */ ticket == nullptr);
		if (f < 0) return -1;
		if (conv_out) {
			edge_out(out_fmt, dst, s->stage, f, s->ch_count, f, s->stream);
			if (take_launch_error()) return -1;
		}
		if (copy_slab(*s, C, out_fmt, out_stride, f, conv_out ? s->stage : dst, nullptr, out)) return -1;
		if (ticket) {
			cudaEvent_t &ev = s->done[t % Shard::DONE_RING];
			if (!ev) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming), return -1);
			CUDA_TRY(cudaEventRecord(ev, s->stream), return -1);
		}
		result = f;
	}
	c->ticket = t;
	if (ticket) *ticket = t;
	return result;
}

long dspb200_chain_submit_host(dspb200_chain *c, long frames, const double *in, double *out, unsigned long long *ticket)
{
	return dspb200_chain_submit_host_io(c, frames, in, DSPB200_IO_F64, 0, out, DSPB200_IO_F64, 0, ticket);
}

int dspb200_chain_wait(dspb200_chain *c, unsigned long long ticket)
{
	if (!c || ticket == 0 || ticket > c->ticket) return -1;
	// A marker is reused every DONE_RING submissions; each shard's stream is in order, so waiting
	// on the newer marker that replaced an old ticket's also covers the old ticket.
	FOR_EACH_SHARD(c, s) {
		cudaEvent_t ev = s->done[ticket % Shard::DONE_RING];
		cudaSetDevice(s->device);
		if (ev) CUDA_TRY(cudaEventSynchronize(ev), return -1);
		else CUDA_TRY(cudaStreamSynchronize(s->stream), return -1);
	}
	if (ticket > c->waited) c->waited = ticket;
	return 0;
}

long dspb200_chain_run_host_io(dspb200_chain *c, long frames, const void *in, int in_fmt, long in_stride, void *out, int out_fmt,
                               long out_stride)
{
	if (!c || !in || !out) return -1;
	if (frames < 1) return 0;
	const long result = dspb200_chain_submit_host_io(c, frames, in, in_fmt, in_stride, out, out_fmt, out_stride, nullptr);
	// also after a failed submit: nothing of this call may still be in flight when we return
	FOR_EACH_SHARD(c, s) {
		cudaSetDevice(s->device);
		CUDA_TRY(cudaStreamSynchronize(s->stream), return -1);
	}
	c->waited = c->ticket;
	return result;
}

long dspb200_chain_run_host(dspb200_chain *c, long frames, const double *in, double *out)
{
	return dspb200_chain_run_host_io(c, frames, in, DSPB200_IO_F64, 0, out, DSPB200_IO_F64, 0);
}

long dspb200_chain_run_device_io(dspb200_chain *c, int shard, long frames, const void *d_in, int in_fmt, long in_stride, void *d_out,
                                 int out_fmt, long out_stride, void *stream)
{
	if (!c || shard < 0 || shard >= (int) c->shards.size() || !d_in || !d_out) return -1;
	if (frames < 1) return 0;
	Shard *s = c->shards[shard].get();
	if (d_in == d_out && !s->ops.empty() && !s->ops.back()->inplace_ok) {
		// checked before anything is enqueued: the operators ahead of the last one would otherwise already have
		// filtered the caller's buffer in place and moved their state on
		set_error("chain: in-place call on a chain whose last operator changes the frame count");
		return -1;
	}
	long max_out = frames;
	s->walk_max_frames(frames, &max_out);
	if (io_refused(in_fmt, in_stride, out_fmt, out_stride, frames, max_out, d_in == d_out)) return -1;
	if (!io_aligned((uintptr_t) d_in, in_fmt) || !io_aligned((uintptr_t) d_out, out_fmt)) {
		set_error("io: a device buffer is not aligned to its element type (%zu bytes in, %zu out)", io_esize(in_fmt), io_esize(out_fmt));
		return -1;
	}
	CUDA_TRY(cudaSetDevice(s->device), return -1);
	if (s->ensure_cap(frames)) return -1;
	cudaStream_t st = (cudaStream_t) stream;   // NULL = the legacy default stream, as everywhere in CUDA
	const bool conv_in = io_kernel(in_fmt) >= 0, conv_out = io_kernel(out_fmt) >= 0;
	if (!conv_in && !conv_out) return s->run_ops(0, frames, (const double *) d_in, (double *) d_out, false, st, false);
	// the edge kernels read d_in and write d_out directly; the operators run on the shard's own buffers in between
	// (buf[0] holds the converted input, and is the result when no operator changes the frame count)
	const double *src = (const double *) d_in;
	if (conv_in) {
		edge_in(in_fmt, d_in, in_stride, s->buf[0], s->ch_count, frames, st);
		if (take_launch_error()) return -1;
		src = s->buf[0];
	}
	bool rate_change = false;
	for (auto &op : s->ops) rate_change |= !op->inplace_ok;
	double *dst = !conv_out ? (double *) d_out : (conv_in && rate_change) ? s->buf[3] : s->buf[0];
	const long f = s->run_ops(0, frames, src, dst, conv_in, st, false);
	if (f < 0) return -1;
	if (conv_out) {
		edge_out(out_fmt, dst, d_out, out_stride, s->ch_count, f, st);
		if (take_launch_error()) return -1;
	}
	return f;
}

long dspb200_chain_run_device(dspb200_chain *c, int shard, long frames, const double *d_in, double *d_out, void *stream)
{
	return dspb200_chain_run_device_io(c, shard, frames, d_in, DSPB200_IO_F64, 0, d_out, DSPB200_IO_F64, 0, stream);
}

int dspb200_chain_join(dspb200_chain *c, int shard, void *stream)
{
	if (!c || shard < 0 || shard >= (int) c->shards.size()) return -1;
	Shard *s = c->shards[shard].get();
	CUDA_TRY(cudaSetDevice(s->device), return -1);
	for (auto &op : s->ops)
		if (op->join((cudaStream_t) stream)) return -1;
	return 0;
}

int dspb200_debug_read(dspb200_chain *c, int shard, int op_index, long long *out, int max)
{
	if (!c || shard < 0 || shard >= (int) c->shards.size() || !out) return -1;
	Shard *s = c->shards[shard].get();
	if (op_index < 0 || op_index >= (int) s->ops.size()) return -1;
	CUDA_TRY(cudaSetDevice(s->device), return -1);
	return s->ops[op_index]->debug_read(out, max);
}

long dspb200_chain_drain_host_io(dspb200_chain *c, long frames, void *out, int out_fmt, long out_stride)
{
	// the drain2 half of drain_effects_chain(), effects_chain.c:1199-1217
	if (!c || !out || frames < 1) return -1;
	const int C = c->channels;
	if (io_refused(IO_F64, 0, out_fmt, out_stride, frames, dspb200_chain_max_out_frames(c, frames), false)) return -2;
	const bool conv_out = io_kernel(out_fmt) >= 0;
	long result = -1;
	FOR_EACH_SHARD(c, s) {
		CUDA_TRY(cudaSetDevice(s->device), return -2);
		if (s->ensure_cap(frames, IO_F64, out_fmt)) return -2;
		long ftmp = frames, dframes = -1;
		size_t idx = 0;
		double *cur = s->buf[0];
		while (idx < s->ops.size() && dframes == -1) {
			Op *op = s->ops[idx].get();
			double *dst = (cur == s->buf[0]) ? s->buf[1] : s->buf[0];
			const long r = op->drain2(ftmp, s->buf[3], dst, s->stream);
			if (r == -2) return -2;
			if (r >= 0) { dframes = r; cur = dst; }
			ftmp = op->max_out_frames(ftmp);
			++idx;
		}
		if (dframes == -1) { result = -1; continue; }
		double *dst = s->buf[3];   // the silence buffer is free again once drain2 has run
		const long f = s->run_ops(idx, dframes, cur, dst, true, s->stream);
		if (f < 0) return -2;
		if (conv_out) {
			edge_out(out_fmt, dst, s->stage, f, s->ch_count, f, s->stream);
			if (take_launch_error()) return -2;
		}
		if (copy_slab(*s, C, out_fmt, out_stride, f, conv_out ? s->stage : dst, nullptr, out)) return -2;
		result = f;
	}
	FOR_EACH_SHARD(c, s) {
		cudaSetDevice(s->device);
		CUDA_TRY(cudaStreamSynchronize(s->stream), return -2);
	}
	return result;
}

long dspb200_chain_drain_host(dspb200_chain *c, long frames, double *out)
{
	return dspb200_chain_drain_host_io(c, frames, out, DSPB200_IO_F64, 0);
}

void dspb200_chain_reset(dspb200_chain *c)
{
	if (!c) return;
	FOR_EACH_SHARD(c, s) {
		cudaSetDevice(s->device);
		for (auto &op : s->ops) op->reset(s->stream);
		cudaStreamSynchronize(s->stream);
	}
}

int dspb200_chain_sync(dspb200_chain *c)
{
	if (!c) return -1;
	FOR_EACH_SHARD(c, s) {
		cudaSetDevice(s->device);
		CUDA_TRY(cudaStreamSynchronize(s->stream), return -1);
	}
	c->waited = c->ticket;
	return 0;
}

int dspb200_hilbert_taps(long taps, double angle, double *h)
{
	// hilbert.c:43-77
	if (taps <= 3 || taps % 2 == 0 || !h) { set_error("hilbert: taps must be odd and > 3"); return -1; }
	const double w_h = sin(-angle), w_d = cos(-angle);
	const long mid = taps / 2;
	for (long i = 0; i < taps; ++i) {
		const long k = i - mid;
		if (k == 0) h[i] = w_d;
		else if (k % 2 == 0) h[i] = 0.0;
		else {
			const double x = 2.0 * M_PI * i / (taps - 1);
			h[i] = w_h * 2.0 / (M_PI * k) * (0.42 - 0.5 * cos(x) + 0.08 * cos(2.0 * x));
		}
	}
	return 0;
}

int dspb200_resample_params(int fs_in, int fs_out, double bandwidth, long out[8])
{
	ResampleParams p;
	if (resample_params_or_error(fs_in, fs_out, bandwidth, &p)) return -1;
	out[0] = p.n; out[1] = p.d; out[2] = p.m; out[3] = p.in_len; out[4] = p.out_len;
	out[5] = p.sinc_len; out[6] = p.out_delay; out[7] = p.in_len;
	return 0;
}

int dspb200_test_rfft(int B, int n_ch, const double *d_in, double *d_spec, void *stream)
{
	if (!g_probe_ok()) return -1;
	return test_rfft(B, n_ch, d_in, d_spec, (cudaStream_t) stream);
}

int dspb200_test_irfft(int B, int n_ch, const double *d_spec, double *d_out2B, void *stream)
{
	if (!g_probe_ok()) return -1;
	return test_irfft(B, n_ch, d_spec, d_out2B, (cudaStream_t) stream);
}

}  // extern "C"
