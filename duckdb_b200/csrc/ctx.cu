// Context, memory and batch staging (host <-> HBM) for libduckdb_b200.
// Replaces: nothing in the reference (it has no device boundary, SURVEY.md section 1); this is the
// "column staging" step 3 of SURVEY.md section 7.
#include "common.cuh"
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <mutex>
#include <unordered_map>
#include <utility>
#include <vector>

static thread_local char g_err[1024] = "";

void b200_set_error(const char *fmt, ...) {
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof(g_err), fmt, ap);
	va_end(ap);
}

int b200_cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
	b200_set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
	if (e == cudaErrorMemoryAllocation) {
		return B200_ERR_OOM;
	}
	if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) {
		return B200_ERR_NO_DEVICE;
	}
	return B200_ERR_CUDA;
}

extern "C" {

const char *b200_last_error(void) {
	return g_err;
}

const char *b200_version(void) {
	return "duckdb_b200 0.1 (sm_90a)";
}

int b200_device_count(void) {
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess) {
		cudaGetLastError();
		return 0;
	}
	return n;
}

int b200_ctx_create(int device, void *stream, b200_ctx **out) {
	if (!out) {
		b200_set_error("b200_ctx_create: out is NULL");
		return B200_ERR_INVALID;
	}
	*out = nullptr;
	int n = b200_device_count();
	if (n <= 0) {
		b200_set_error("b200_ctx_create: no CUDA device available (there is no CPU fallback)");
		return B200_ERR_NO_DEVICE;
	}
	if (device < 0 || device >= n) {
		b200_set_error("b200_ctx_create: device %d out of range (%d devices)", device, n);
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(device));
	b200_ctx *ctx = new b200_ctx();
	ctx->device = device;
	ctx->launches = ctx->h2d_bytes = ctx->d2h_bytes = 0;
	if (stream) {
		ctx->stream = (cudaStream_t)stream;
		ctx->own_stream = false;
	} else {
		cudaError_t e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
		if (e != cudaSuccess) {
			delete ctx;
			return b200_cuda_fail(e, "cudaStreamCreate", __FILE__, __LINE__);
		}
		ctx->own_stream = true;
	}
	ctx->pinned_scratch = nullptr;
	ctx->dev_scratch = nullptr;
	ctx->sm_count = B200_SM_COUNT;
	{
		int sms = 0;
		if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0) {
			ctx->sm_count = sms;
		}
	}
	// keep freed blocks cached in the pool: operators re-allocate the same sizes every batch
	cudaMemPool_t pool;
	if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
		uint64_t thresh = UINT64_MAX;
		cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh);
	}
	// experiment knob: B200_L2_FETCH=32|64|128 sets cudaLimitMaxL2FetchGranularity (the default is left alone)
	{
		const char *env = getenv("B200_L2_FETCH");
		if (env && atoi(env) > 0) {
			cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(env));
			cudaGetLastError();
		}
	}
	// set aside the maximum persisting L2 carve-out (used for join / aggregate tables, see b200_l2_pin)
	{
		int v = 0;
		ctx->l2_persist_max = ctx->l2_window_max = 0;
		ctx->l2_size = (size_t)50 << 20;
		if (cudaDeviceGetAttribute(&v, cudaDevAttrL2CacheSize, device) == cudaSuccess && v > 0) {
			ctx->l2_size = (size_t)v;
		}
		if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxPersistingL2CacheSize, device) == cudaSuccess && v > 0) {
			ctx->l2_persist_max = (size_t)v;
		}
		if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxAccessPolicyWindowSize, device) == cudaSuccess && v > 0) {
			ctx->l2_window_max = (size_t)v;
		}
		cudaGetLastError();
		// Opt-in (B200_L2_PIN=1).  The lean probe kernels read their input with evict-first streaming loads, and the
		// carve-out survives the operator in ways the runtime does not undo reliably, so it can slow down the
		// operators that run after a pinned probe in the same process.
		if (!getenv("B200_L2_PIN") || getenv("B200_NO_L2_PIN")) {
			ctx->l2_persist_max = 0;
		}
	}
	cudaError_t e = cudaHostAlloc((void **)&ctx->pinned_scratch, 64 * sizeof(uint64_t), cudaHostAllocDefault);
	e = e ? e : cudaMalloc((void **)&ctx->dev_scratch, 64 * sizeof(uint64_t));
	if (e != cudaSuccess) {
		int rc = b200_cuda_fail(e, "context scratch allocation", __FILE__, __LINE__);
		b200_ctx_destroy(ctx);
		return rc;
	}
	*out = ctx;
	return B200_OK;
}

void b200_ctx_destroy(b200_ctx *ctx) {
	if (!ctx) {
		return;
	}
	cudaSetDevice(ctx->device);
	cudaStreamSynchronize(ctx->stream);
	if (ctx->pinned_scratch) {
		cudaFreeHost(ctx->pinned_scratch);
	}
	if (ctx->dev_scratch) {
		cudaFree(ctx->dev_scratch);
	}
	if (ctx->own_stream) {
		cudaStreamDestroy(ctx->stream);
	}
	delete ctx;
}

int b200_ctx_sync(b200_ctx *ctx) {
	if (!ctx) {
		b200_set_error("b200_ctx_sync: ctx is NULL");
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaStreamSynchronize(ctx->stream));
	return B200_OK;
}

int b200_ctx_stats(b200_ctx *ctx, uint64_t *launches, uint64_t *h2d, uint64_t *d2h) {
	if (!ctx) {
		return B200_ERR_INVALID;
	}
	if (launches) {
		*launches = ctx->launches;
	}
	if (h2d) {
		*h2d = ctx->h2d_bytes;
	}
	if (d2h) {
		*d2h = ctx->d2h_bytes;
	}
	return B200_OK;
}

// Pinned staging memory is expensive to create (page-locking runs at a few GB/s: the 16 workers x 2 morsel buffers of a
// DuckDB query are ~1 s of cudaHostAlloc) and cheap to keep, so released buffers go to a process-wide cache (bounded by
// B200_HOST_CACHE_MB, default 8192) and b200_host_alloc re-uses a cached buffer of at least - and at most twice - the
// requested size.  b200_host_trim() returns the cache to the OS.
static std::mutex g_host_mu;
static std::unordered_map<void *, size_t> g_host_size;        // every live or cached buffer -> its real size
static std::vector<std::pair<size_t, void *>> g_host_cache;   // released buffers
static size_t g_host_cached_bytes = 0;

int b200_host_alloc(b200_ctx *ctx, size_t bytes, void **out) {
	if (!ctx || !out) {
		return B200_ERR_INVALID;
	}
	const size_t want = ((bytes ? bytes : 1) + ((size_t)1 << 20) - 1) & ~(((size_t)1 << 20) - 1);
	{
		std::lock_guard<std::mutex> guard(g_host_mu);
		size_t best = g_host_cache.size();
		for (size_t i = 0; i < g_host_cache.size(); i++) {
			if (g_host_cache[i].first >= want && g_host_cache[i].first <= 2 * want &&
			    (best == g_host_cache.size() || g_host_cache[i].first < g_host_cache[best].first)) {
				best = i;
			}
		}
		if (best != g_host_cache.size()) {
			*out = g_host_cache[best].second;
			g_host_cached_bytes -= g_host_cache[best].first;
			g_host_cache.erase(g_host_cache.begin() + best);
			return B200_OK;
		}
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	CUDA_TRY(cudaHostAlloc(out, want, cudaHostAllocPortable));
	std::lock_guard<std::mutex> guard(g_host_mu);
	g_host_size[*out] = want;
	return B200_OK;
}

int b200_host_free(b200_ctx *ctx, void *ptr) {
	(void)ctx;
	if (!ptr) {
		return B200_OK;
	}
	static const size_t limit = (size_t)(getenv("B200_HOST_CACHE_MB") ? atoll(getenv("B200_HOST_CACHE_MB")) : 8192) << 20;
	{
		std::lock_guard<std::mutex> guard(g_host_mu);
		auto it = g_host_size.find(ptr);
		if (it != g_host_size.end() && g_host_cached_bytes + it->second <= limit) {
			g_host_cache.emplace_back(it->second, ptr);
			g_host_cached_bytes += it->second;
			return B200_OK;
		}
		if (it != g_host_size.end()) {
			g_host_size.erase(it);
		}
	}
	CUDA_TRY(cudaFreeHost(ptr));
	return B200_OK;
}

int b200_host_trim(void) {
	std::vector<std::pair<size_t, void *>> drop;
	{
		std::lock_guard<std::mutex> guard(g_host_mu);
		drop.swap(g_host_cache);
		g_host_cached_bytes = 0;
		for (auto &e : drop) {
			g_host_size.erase(e.second);
		}
	}
	for (auto &e : drop) {
		CUDA_TRY(cudaFreeHost(e.second));
	}
	return B200_OK;
}

} // extern "C"

void b200_l2_pin(b200_ctx *ctx, const void *ptr, size_t bytes) {
	if (!ctx->l2_persist_max || !ctx->l2_window_max || !ptr || !bytes) {
		return;
	}
	cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, ctx->l2_persist_max); // carve-out only while a table is pinned
	cudaStreamAttrValue attr;
	memset(&attr, 0, sizeof(attr));
	size_t win = bytes < ctx->l2_window_max ? bytes : ctx->l2_window_max;
	attr.accessPolicyWindow.base_ptr = const_cast<void *>(ptr);
	attr.accessPolicyWindow.num_bytes = win;
	double ratio = (double)ctx->l2_persist_max / (double)win;
	attr.accessPolicyWindow.hitRatio = ratio > 1.0 ? 1.0f : (float)ratio;
	attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
	attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
	cudaStreamSetAttribute(ctx->stream, cudaStreamAttributeAccessPolicyWindow, &attr);
	cudaGetLastError();
}

void b200_l2_unpin(b200_ctx *ctx) {
	if (!ctx->l2_persist_max || !ctx->l2_window_max) {
		return;
	}
	cudaStreamAttrValue attr;
	memset(&attr, 0, sizeof(attr));
	attr.accessPolicyWindow.num_bytes = 0;
	cudaStreamSetAttribute(ctx->stream, cudaStreamAttributeAccessPolicyWindow, &attr);
	// give the persisting lines AND the carve-out back: a standing carve-out / stale persisting lines slow the next
	// operator down
	if (!getenv("B200_L2_KEEP")) {
		cudaCtxResetPersistingL2Cache();
		cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, 0);
	}
	cudaGetLastError();
}

int b200_dev_alloc(b200_ctx *ctx, size_t bytes, void **out) {
	if (bytes == 0) {
		bytes = 16;
	}
	cudaError_t e = cudaMallocAsync(out, bytes, ctx->stream);
	if (e != cudaSuccess) {
		*out = nullptr;
		return b200_cuda_fail(e, "cudaMallocAsync", __FILE__, __LINE__);
	}
	return B200_OK;
}

void b200_dev_free(b200_ctx *ctx, void *p) {
	if (p) {
		cudaFreeAsync(p, ctx->stream);
	}
}

b200_batch *b200_batch_new(b200_ctx *ctx, uint64_t nrows) {
	b200_batch *b = new b200_batch();
	b->ctx = ctx;
	b->nrows = nrows;
	return b;
}

int b200_batch_add_flat(b200_batch *b, int type, uint64_t capacity_rows, bool with_validity, void **data,
                        uint64_t **validity) {
	int sz = b200_type_size(type);
	if (!sz) {
		b200_set_error("unsupported column type %d", type);
		return B200_ERR_INVALID;
	}
	void *d = nullptr;
	B200_TRY(b200_dev_alloc(b->ctx, (size_t)capacity_rows * sz + 16, &d));
	b->owned.push_back(d);
	uint64_t *v = nullptr;
	if (with_validity) {
		size_t words = (capacity_rows + 63) / 64 + 1;
		void *vp = nullptr;
		B200_TRY(b200_dev_alloc(b->ctx, words * 8, &vp));
		b->owned.push_back(vp);
		v = (uint64_t *)vp;
	}
	DCol c;
	c.data = d;
	c.sel = nullptr;
	c.validity = v;
	c.type = type;
	c.vtype = B200_FLAT_VECTOR;
	b->cols.push_back(c);
	b->dict_sizes.push_back(0);
	if (data) {
		*data = d;
	}
	if (validity) {
		*validity = v;
	}
	return B200_OK;
}

static int check_vector(const b200_vector &v, int i, uint64_t nrows) {
	if (!b200_type_size(v.type)) {
		b200_set_error("column %d: unsupported type %d", i, v.type);
		return B200_ERR_INVALID;
	}
	if (v.vector_type != B200_FLAT_VECTOR && v.vector_type != B200_CONSTANT_VECTOR &&
	    v.vector_type != B200_DICTIONARY_VECTOR) {
		b200_set_error("column %d: unsupported vector type %d", i, v.vector_type);
		return B200_ERR_INVALID;
	}
	if (v.vector_type == B200_DICTIONARY_VECTOR && !v.sel) {
		b200_set_error("column %d: dictionary vector without selection", i);
		return B200_ERR_INVALID;
	}
	if (!v.data && !(nrows == 0 && v.vector_type == B200_FLAT_VECTOR)) { // an empty flat column may have no buffer
		b200_set_error("column %d: data is NULL", i);
		return B200_ERR_INVALID;
	}
	return B200_OK;
}

extern "C" {

int b200_batch_upload(b200_ctx *ctx, const b200_vector *cols, int ncols, uint64_t nrows, b200_batch **out) {
	if (!ctx || !out || (ncols > 0 && !cols) || ncols < 0) {
		b200_set_error("b200_batch_upload: bad arguments");
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	for (int i = 0; i < ncols; i++) {
		B200_TRY(check_vector(cols[i], i, nrows));
	}
	b200_batch *b = b200_batch_new(ctx, nrows);
	for (int i = 0; i < ncols; i++) {
		const b200_vector &v = cols[i];
		int sz = b200_type_size(v.type);
		uint64_t nvals = v.vector_type == B200_FLAT_VECTOR       ? nrows
		                 : v.vector_type == B200_CONSTANT_VECTOR ? 1
		                                                         : v.dict_size;
		DCol c;
		c.type = v.type;
		c.vtype = v.vector_type;
		c.sel = nullptr;
		c.validity = nullptr;
		void *d = nullptr;
		size_t bytes = (size_t)nvals * sz;
		int r = b200_dev_alloc(ctx, bytes + 16, &d);
		if (r != B200_OK) {
			b200_batch_free(b);
			return r;
		}
		b->owned.push_back(d);
		if (bytes) {
			cudaError_t e = cudaMemcpyAsync(d, v.data, bytes, cudaMemcpyHostToDevice, ctx->stream);
			if (e != cudaSuccess) {
				b200_batch_free(b);
				return b200_cuda_fail(e, "cudaMemcpyAsync(H2D data)", __FILE__, __LINE__);
			}
			ctx->h2d_bytes += bytes;
		}
		c.data = d;
		if (v.validity) {
			size_t vbytes = ((nvals + 63) / 64) * 8;
			void *vp = nullptr;
			r = b200_dev_alloc(ctx, vbytes + 16, &vp);
			if (r != B200_OK) {
				b200_batch_free(b);
				return r;
			}
			b->owned.push_back(vp);
			if (vbytes) {
				cudaError_t e = cudaMemcpyAsync(vp, v.validity, vbytes, cudaMemcpyHostToDevice, ctx->stream);
				if (e != cudaSuccess) {
					b200_batch_free(b);
					return b200_cuda_fail(e, "cudaMemcpyAsync(H2D validity)", __FILE__, __LINE__);
				}
				ctx->h2d_bytes += vbytes;
			}
			c.validity = (const uint64_t *)vp;
		}
		if (v.vector_type == B200_DICTIONARY_VECTOR) {
			size_t sbytes = (size_t)nrows * 4;
			void *sp = nullptr;
			r = b200_dev_alloc(ctx, sbytes + 16, &sp);
			if (r != B200_OK) {
				b200_batch_free(b);
				return r;
			}
			b->owned.push_back(sp);
			if (sbytes) {
				cudaError_t e = cudaMemcpyAsync(sp, v.sel, sbytes, cudaMemcpyHostToDevice, ctx->stream);
				if (e != cudaSuccess) {
					b200_batch_free(b);
					return b200_cuda_fail(e, "cudaMemcpyAsync(H2D sel)", __FILE__, __LINE__);
				}
				ctx->h2d_bytes += sbytes;
			}
			c.sel = (const uint32_t *)sp;
		}
		b->cols.push_back(c);
		b->dict_sizes.push_back(v.dict_size);
	}
	*out = b;
	return B200_OK;
}

// Upload into device buffers the CALLER owns (a worker's persistent device ring): no allocation on the row path, the
// copies are asynchronous on the context's stream, the batch only references the buffers.
int b200_batch_upload_to(b200_ctx *ctx, const b200_vector *cols, int ncols, uint64_t nrows, void *const *dev_data,
                         void *const *dev_validity, b200_batch **out) {
	if (!ctx || !out || ncols < 0 || (ncols > 0 && (!cols || !dev_data))) {
		b200_set_error("b200_batch_upload_to: bad arguments");
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	for (int i = 0; i < ncols; i++) {
		B200_TRY(check_vector(cols[i], i, nrows));
		if (cols[i].vector_type != B200_FLAT_VECTOR || !dev_data[i] || (cols[i].validity && (!dev_validity || !dev_validity[i]))) {
			b200_set_error("b200_batch_upload_to: column %d must be a flat vector with a device buffer (and a validity buffer "
			               "when it has a validity mask)", i);
			return B200_ERR_INVALID;
		}
	}
	b200_batch *b = b200_batch_new(ctx, nrows);
	for (int i = 0; i < ncols; i++) {
		const b200_vector &v = cols[i];
		DCol c;
		c.type = v.type;
		c.vtype = B200_FLAT_VECTOR;
		c.sel = nullptr;
		c.validity = nullptr;
		c.data = dev_data[i];
		size_t bytes = (size_t)nrows * b200_type_size(v.type);
		cudaError_t e = bytes ? cudaMemcpyAsync(dev_data[i], v.data, bytes, cudaMemcpyHostToDevice, ctx->stream) : cudaSuccess;
		if (e == cudaSuccess && v.validity) {
			size_t vbytes = ((nrows + 63) / 64) * 8;
			e = vbytes ? cudaMemcpyAsync(dev_validity[i], v.validity, vbytes, cudaMemcpyHostToDevice, ctx->stream) : cudaSuccess;
			c.validity = (const uint64_t *)dev_validity[i];
			ctx->h2d_bytes += vbytes;
		}
		if (e != cudaSuccess) {
			b200_batch_free(b);
			return b200_cuda_fail(e, "cudaMemcpyAsync(H2D, caller's device buffer)", __FILE__, __LINE__);
		}
		ctx->h2d_bytes += bytes;
		b->cols.push_back(c);
		b->dict_sizes.push_back(0);
	}
	*out = b;
	return B200_OK;
}

int b200_batch_wrap(b200_ctx *ctx, const b200_vector *cols, int ncols, uint64_t nrows, b200_batch **out) {
	if (!ctx || !out || (ncols > 0 && !cols) || ncols < 0) {
		b200_set_error("b200_batch_wrap: bad arguments");
		return B200_ERR_INVALID;
	}
	for (int i = 0; i < ncols; i++) {
		B200_TRY(check_vector(cols[i], i, nrows));
	}
	b200_batch *b = b200_batch_new(ctx, nrows);
	for (int i = 0; i < ncols; i++) {
		DCol c;
		c.type = cols[i].type;
		c.vtype = cols[i].vector_type;
		c.data = cols[i].data;
		c.sel = cols[i].sel;
		c.validity = cols[i].validity;
		b->cols.push_back(c);
		b->dict_sizes.push_back(cols[i].dict_size);
	}
	*out = b;
	return B200_OK;
}

uint64_t b200_batch_rows(const b200_batch *b) {
	return b ? b->nrows : 0;
}

int b200_batch_cols(const b200_batch *b) {
	return b ? (int)b->cols.size() : 0;
}

int b200_batch_column(const b200_batch *b, int col, b200_vector *out) {
	if (!b || !out || col < 0 || col >= (int)b->cols.size()) {
		b200_set_error("b200_batch_column: bad arguments");
		return B200_ERR_INVALID;
	}
	const DCol &c = b->cols[col];
	out->type = c.type;
	out->vector_type = c.vtype;
	out->data = c.data;
	out->sel = c.sel;
	out->validity = c.validity;
	out->dict_size = b->dict_sizes[col];
	return B200_OK;
}

int b200_batch_download(b200_ctx *ctx, const b200_batch *b, int col, void *dst_data, uint64_t *dst_validity) {
	if (!ctx || !b || col < 0 || col >= (int)b->cols.size()) {
		b200_set_error("b200_batch_download: bad arguments");
		return B200_ERR_INVALID;
	}
	const DCol &c = b->cols[col];
	if (c.vtype != B200_FLAT_VECTOR) {
		b200_set_error("b200_batch_download: only flat columns can be downloaded");
		return B200_ERR_INVALID;
	}
	CUDA_TRY(cudaSetDevice(ctx->device));
	size_t bytes = (size_t)b->nrows * b200_type_size(c.type);
	if (dst_data && bytes) {
		CUDA_TRY(cudaMemcpyAsync(dst_data, c.data, bytes, cudaMemcpyDeviceToHost, ctx->stream));
		ctx->d2h_bytes += bytes;
	}
	if (dst_validity) {
		size_t words = (b->nrows + 63) / 64;
		if (c.validity) {
			if (words) {
				CUDA_TRY(
				    cudaMemcpyAsync(dst_validity, c.validity, words * 8, cudaMemcpyDeviceToHost, ctx->stream));
				ctx->d2h_bytes += words * 8;
			}
		} else {
			// all valid; order after any pending async copies into the same buffer
			CUDA_TRY(cudaStreamSynchronize(ctx->stream));
			memset(dst_validity, 0xff, words * 8);
		}
	}
	CUDA_TRY(cudaStreamSynchronize(ctx->stream));
	return B200_OK;
}

void b200_batch_free(b200_batch *b) {
	if (!b) {
		return;
	}
	cudaSetDevice(b->ctx->device);
	for (void *p : b->owned) {
		b200_dev_free(b->ctx, p);
	}
	delete b;
}

} // extern "C"
