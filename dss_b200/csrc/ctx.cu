// ctx.cu -- context lifetime, error strings, grow-only scratch, single-pass exclusive scan.
#include <stdarg.h>
#include <stdlib.h>

#include "common.cuh"

namespace dss {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int ctx_reserve(dss_ctx *ctx, BufId id, size_t bytes, void **out) {
    if (bytes < 256) bytes = 256;
    if (ctx->cap[id] < bytes) {
        // grow geometrically; cudaFree waits for kernels still using the old block
        size_t want = bytes + bytes / 2;
        want = (want + 255) & ~size_t(255);
        if (ctx->buf[id]) {
            cudaFree(ctx->buf[id]);
            ctx->buf[id] = nullptr;
            ctx->cap[id] = 0;
        }
        void *p = nullptr;
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) {
            cudaGetLastError();
            e = cudaMalloc(&p, bytes);  // retry without the slack
            want = bytes;
        }
        if (e != cudaSuccess) {
            cudaGetLastError();
            set_error("scratch allocation of %zu bytes failed: %s", bytes, cudaGetErrorString(e));
            return DSS_E_NOMEM;
        }
        ctx->buf[id] = p;
        ctx->cap[id] = want;
    }
    *out = ctx->buf[id];
    return DSS_OK;
}

void prof_begin(dss_ctx *ctx, int stage, cudaStream_t st) {
    // scopes may nest (e.g. the scan inside the occupancy backward): keep a small stack of open entries
    if (ctx->n_open >= 8) {
        ctx->open[ctx->n_open++ & 7] = -1;
        return;
    }
    if (ctx->n_pending == ctx->cap_pending) {
        const int ncap = ctx->cap_pending ? ctx->cap_pending * 2 : 256;
        ProfPending *np = (ProfPending *)realloc(ctx->pending, sizeof(ProfPending) * ncap);
        if (!np) {
            ctx->open[ctx->n_open++] = -1;
            return;
        }
        for (int i = ctx->cap_pending; i < ncap; ++i) {
            np[i].a = nullptr;
            np[i].b = nullptr;
        }
        ctx->pending = np;
        ctx->cap_pending = ncap;
    }
    const int slot = ctx->n_pending++;
    ProfPending &p = ctx->pending[slot];
    if (!p.a) cudaEventCreate(&p.a);
    if (!p.b) cudaEventCreate(&p.b);
    p.stage = stage;
    p.closed = 0;
    cudaEventRecord(p.a, st);
    ctx->open[ctx->n_open++] = slot;
}

void prof_end(dss_ctx *ctx, cudaStream_t st) {
    if (ctx->n_open <= 0) return;
    const int slot = ctx->open[--ctx->n_open & 7];
    if (slot < 0) return;
    cudaEventRecord(ctx->pending[slot].b, st);
    ctx->pending[slot].closed = 1;
}

static void prof_collect(dss_ctx *ctx) {
    for (int i = 0; i < ctx->n_pending; ++i) {
        ProfPending &p = ctx->pending[i];
        float ms = 0.f;
        if (!p.closed) continue;
        if (cudaEventSynchronize(p.b) == cudaSuccess && cudaEventElapsedTime(&ms, p.a, p.b) == cudaSuccess) {
            ctx->stage_ms[p.stage] += ms;
            ctx->stage_calls[p.stage] += 1;
        } else {
            cudaGetLastError();
        }
    }
    ctx->n_pending = 0;
    ctx->n_open = 0;
}

static const char *k_stage_names[NUM_STAGES] = {
    "pack_records", "preprocess", "bin_count", "scan", "bin_scatter", "raster_forward", "visibility",
    "search_radius", "occ_backward", "colour_backward", "zbuf_backward", "chain_world", "grid_2d", "occ_bin", "knn",
    "camera_backward", "light_backward", "depth_forward", "depth_backward"};

// ---------------------------------------------------------------------------------------------
// Exclusive scan, single pass with decoupled look-back.  Replaces external/prefix_sum
// (Blelloch + recursion + cudaMalloc/cudaFree per level: prefix_sum.cu:135-205).
// One tile = 256 threads x 8 items.  status word: [63:32] flag (0 none, 1 aggregate, 2 inclusive),
// [31:0] value.  Tiles are claimed through an atomic ticket so look-back never waits on a tile
// that has not started.
// ---------------------------------------------------------------------------------------------
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__global__ void __launch_bounds__(SCAN_THREADS)
scan_kernel(const int32_t *in, int32_t *out, int64_t n, unsigned long long *status,
            unsigned int *ticket) {
    __shared__ int32_t s_data[SCAN_TILE];
    __shared__ int32_t s_warp[SCAN_THREADS / 32];
    __shared__ unsigned int s_tile;
    __shared__ int32_t s_prefix;

    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const unsigned int tile = s_tile;
    const int64_t base = (int64_t)tile * SCAN_TILE;

    // coalesced (striped) load into shared memory
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        const int o = j * SCAN_THREADS + threadIdx.x;
        const int64_t g = base + o;
        s_data[o] = (g < n) ? in[g] : 0;
    }
    __syncthreads();

    // each thread scans 8 consecutive items (blocked arrangement)
    int32_t v[SCAN_ITEMS];
    int32_t sum = 0;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        v[j] = s_data[threadIdx.x * SCAN_ITEMS + j];
        sum += v[j];
    }
    // block-wide exclusive scan of per-thread sums
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int32_t incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int32_t w = (lane < SCAN_THREADS / 32) ? s_warp[lane] : 0;
#pragma unroll
        for (int d = 1; d < SCAN_THREADS / 32; d <<= 1) {
            const int32_t t = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += t;
        }
        if (lane < SCAN_THREADS / 32) s_warp[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    const int32_t warp_excl = (warp == 0) ? 0 : s_warp[warp - 1];
    const int32_t thread_excl = warp_excl + incl - sum;
    const int32_t tile_total = s_warp[SCAN_THREADS / 32 - 1];

    // publish aggregate / look back (warp 0)
    if (warp == 0) {
        if (tile == 0) {
            if (lane == 0) {
                atomicExch(&status[0], (2ull << 32) | (unsigned int)tile_total);
                s_prefix = 0;
            }
        } else {
            if (lane == 0) atomicExch(&status[tile], (1ull << 32) | (unsigned int)tile_total);
            int32_t running = 0;
            int64_t look = (int64_t)tile - 1;
            while (true) {
                const int64_t t = look - lane;
                unsigned long long s = (2ull << 32);  // tiles before 0 act as inclusive zero
                if (t >= 0) {
                    do {
                        s = *((volatile unsigned long long *)&status[t]);
                    } while ((s >> 32) == 0ull);
                }
                const unsigned int flag = (unsigned int)(s >> 32);
                const int32_t val = (int32_t)(unsigned int)(s & 0xffffffffull);
                // first lane (closest tile is lane 0) that holds an inclusive prefix terminates the walk
                const unsigned int incl_mask = __ballot_sync(0xffffffffu, flag == 2u);
                int32_t contrib = val;
                if (incl_mask) {
                    const int first = __ffs(incl_mask) - 1;
                    if (lane > first) contrib = 0;
                }
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, d);
                running += contrib;
                if (incl_mask) break;
                look -= 32;
            }
            if (lane == 0) {
                atomicExch(&status[tile], (2ull << 32) | (unsigned int)(running + tile_total));
                s_prefix = running;
            }
        }
    }
    __syncthreads();
    const int32_t prefix = s_prefix;

    int32_t run = prefix + thread_excl;
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        s_data[threadIdx.x * SCAN_ITEMS + j] = run;
        run += v[j];
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < SCAN_ITEMS; ++j) {
        const int o = j * SCAN_THREADS + threadIdx.x;
        const int64_t g = base + o;
        if (g < n) out[g] = s_data[o];
    }
}

__global__ void publish_words_kernel(const uint32_t *__restrict__ src, uint32_t *dst, int n) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
    __threadfence_system();
}

int publish_words(dss_ctx *ctx, const void *src_device, void *dst_pinned_host, int n_words, cudaStream_t st) {
    if (n_words <= 0) return DSS_OK;
    void *dst_dev = nullptr;
    DSS_CUDA_TRY(cudaHostGetDevicePointer(&dst_dev, dst_pinned_host, 0));
    publish_words_kernel<<<1, 128, 0, st>>>(reinterpret_cast<const uint32_t *>(src_device),
                                           reinterpret_cast<uint32_t *>(dst_dev), n_words);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

int exclusive_scan_i32(dss_ctx *ctx, const int32_t *in, int32_t *out, int64_t n, cudaStream_t st) {
    if (n <= 0) return DSS_OK;
    const int64_t tiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    unsigned long long *status = nullptr;
    int rc = ctx_get(ctx, BUF_SCAN_STATUS, (size_t)tiles + 1, &status);
    if (rc) return rc;
    DSS_CUDA_TRY(cudaMemsetAsync(status, 0, ((size_t)tiles + 1) * sizeof(unsigned long long), st));
    unsigned int *ticket = reinterpret_cast<unsigned int *>(status + tiles);
    StageScope prof(ctx, ST_SCAN, st);
    scan_kernel<<<(unsigned int)tiles, SCAN_THREADS, 0, st>>>(in, out, n, status, ticket);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

// ---------------------------------------------------------------------------------------------
// 64-bit exclusive scan in place, three launches: per-tile sums, one block scanning the tile sums (and writing the
// grand total to v[n]), then each tile applied from its carry.  Integer sums, so the result does not depend on the
// order of anything.  Used by the mesh rasterizer (pixel items per (view, face)) and the Poisson-disk sampler (face
// weights).
// ---------------------------------------------------------------------------------------------

// exclusive scan of v over the block (SCAN_THREADS threads); returns the block total through `total`
__device__ __forceinline__ int64_t block_exclusive_scan_i64(int64_t v, int64_t &total) {
    __shared__ int64_t sWarp[SCAN_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int64_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
    }
    if (lane == 31) sWarp[warp] = inc;
    __syncthreads();
    int64_t before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < SCAN_THREADS / 32; ++w) {
        if (w < warp) before += sWarp[w];
        total += sWarp[w];
    }
    __syncthreads();
    return before + inc - v;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_i64_tiles_kernel(const int64_t *v, int64_t n,
                                                                      int64_t *tile_sums) {
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
    int64_t s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) s += base + k < n ? v[base + k] : 0;
    int64_t total;
    block_exclusive_scan_i64(s, total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

// one block: exclusive scan of the tile sums in place; the grand total goes to v[n]
__global__ void __launch_bounds__(SCAN_THREADS) scan_i64_sums_kernel(int64_t *tile_sums, int64_t tiles, int64_t *v,
                                                                     int64_t n) {
    int64_t carry = 0;
    for (int64_t b0 = 0; b0 < tiles; b0 += SCAN_THREADS) {
        const int64_t b = b0 + threadIdx.x;
        const int64_t x = b < tiles ? tile_sums[b] : 0;
        int64_t total;
        const int64_t ex = block_exclusive_scan_i64(x, total);
        if (b < tiles) tile_sums[b] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) v[n] = carry;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_i64_apply_kernel(int64_t *v, int64_t n,
                                                                      const int64_t *tile_sums) {
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * SCAN_ITEMS;
    int64_t x[SCAN_ITEMS], s = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        x[k] = base + k < n ? v[base + k] : 0;
        s += x[k];
    }
    int64_t total;
    int64_t run = tile_sums[blockIdx.x] + block_exclusive_scan_i64(s, total);
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
        if (base + k < n) v[base + k] = run;
        run += x[k];
    }
}

int64_t scan_i64_tiles(int64_t n) { return (n + SCAN_TILE - 1) / SCAN_TILE; }

int exclusive_scan_i64(dss_ctx *ctx, int64_t *v, int64_t n, int64_t *tile_sums, cudaStream_t st) {
    if (n <= 0) return DSS_OK;
    const int64_t tiles = scan_i64_tiles(n);
    scan_i64_tiles_kernel<<<(unsigned int)tiles, SCAN_THREADS, 0, st>>>(v, n, tile_sums);
    DSS_LAUNCH_CHECK(ctx);
    scan_i64_sums_kernel<<<1, SCAN_THREADS, 0, st>>>(tile_sums, tiles, v, n);
    DSS_LAUNCH_CHECK(ctx);
    scan_i64_apply_kernel<<<(unsigned int)tiles, SCAN_THREADS, 0, st>>>(v, n, tile_sums);
    DSS_LAUNCH_CHECK(ctx);
    return DSS_OK;
}

}  // namespace dss

extern "C" {

int dss_version(void) { return 1; }

const char *dss_last_error(void) { return dss::g_err; }

int dss_create(dss_ctx **out) {
    DSS_REQUIRE(out != nullptr, "out pointer is null");
    int dev = 0;
    DSS_CUDA_TRY(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    DSS_CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code loads on compute capability 9.0 only
        dss::set_error("libdss_b200 is built for sm_90a only; device %d is sm_%d%d", dev, prop.major,
                       prop.minor);
        return DSS_E_CUDA;
    }
    dss_ctx *c = new dss_ctx();
    memset(c, 0, sizeof(*c));
    c->device = dev;
    c->sm_count = prop.multiProcessorCount;
    {
        const char *e = getenv("DSS_BIN_DIRECT");
        c->bin_direct = (e && e[0] == '1') ? 1 : 0;
        const char *nr = getenv("DSS_BIN_NORECTS");
        c->bin_no_rects = (nr && nr[0] == '1') ? 1 : 0;
        const char *mb = getenv("DSS_RASTER_MINB");
        c->raster_minb5 = (mb && mb[0] == '5') ? 1 : 0;
        const char *sf = getenv("DSS_SYNC_FORWARD");
        c->sync_forward = (sf && sf[0] == '1') ? 1 : 0;
        const char *to = getenv("DSS_NO_TILE_ORDER");
        c->no_tile_order = (to && to[0] == '1') ? 1 : 0;
        const char *ns = getenv("DSS_NS");
        c->ns_override = ns ? atoi(ns) : 0;
    }
    if (cudaHostAlloc((void **)&c->h_pinned, 64 * sizeof(int64_t), cudaHostAllocMapped) != cudaSuccess) {
        cudaGetLastError();
        delete c;
        dss::set_error("pinned host allocation failed");
        return DSS_E_NOMEM;
    }
    memset(c->h_pinned, 0, 64 * sizeof(int64_t));
    if (cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking) != cudaSuccess) {
        cudaGetLastError();
        cudaFreeHost(c->h_pinned);
        delete c;
        dss::set_error("event creation failed");
        return DSS_E_CUDA;
    }
    *out = c;
    return DSS_OK;
}

void dss_destroy(dss_ctx *ctx) {
    if (!ctx) return;
    for (int i = 0; i < ctx->cap_pending; ++i) {
        if (ctx->pending[i].a) cudaEventDestroy(ctx->pending[i].a);
        if (ctx->pending[i].b) cudaEventDestroy(ctx->pending[i].b);
    }
    free(ctx->pending);
    for (int i = 0; i < dss::NUM_BUFS; ++i)
        if (ctx->buf[i]) cudaFree(ctx->buf[i]);
    if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    if (ctx->side) cudaStreamDestroy(ctx->side);
    delete ctx;
}

size_t dss_scratch_bytes(const dss_ctx *ctx) {
    size_t s = 0;
    if (ctx)
        for (int i = 0; i < dss::NUM_BUFS; ++i) s += ctx->cap[i];
    return s;
}

int64_t dss_launch_count(const dss_ctx *ctx) { return ctx ? ctx->launches : 0; }

int dss_profile_enable(dss_ctx *ctx, int on) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    if (!on && ctx->profiling) dss::prof_collect(ctx);
    ctx->profiling = on ? 1 : 0;
    return DSS_OK;
}

int dss_profile_reset(dss_ctx *ctx) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    dss::prof_collect(ctx);
    for (int i = 0; i < dss::NUM_STAGES; ++i) {
        ctx->stage_ms[i] = 0.0;
        ctx->stage_calls[i] = 0;
    }
    return DSS_OK;
}

int dss_profile_num_stages(void) { return dss::NUM_STAGES; }

const char *dss_profile_stage_name(int stage) {
    return (stage >= 0 && stage < dss::NUM_STAGES) ? dss::k_stage_names[stage] : "";
}

int dss_profile_read(dss_ctx *ctx, int stage, double *total_ms, int64_t *brackets) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(stage >= 0 && stage < dss::NUM_STAGES, "stage out of range");
    dss::prof_collect(ctx);
    if (total_ms) *total_ms = ctx->stage_ms[stage];
    if (brackets) *brackets = ctx->stage_calls[stage];
    return DSS_OK;
}

int dss_exclusive_scan_i32(dss_ctx *ctx, const int32_t *in, int32_t *out, int64_t n, void *stream) {
    DSS_REQUIRE(ctx != nullptr, "ctx is null");
    DSS_REQUIRE(n >= 0, "n must be non-negative");
    if (n == 0) return DSS_OK;
    DSS_REQUIRE(in != nullptr && out != nullptr, "null array");
    return dss::exclusive_scan_i32(ctx, in, out, n, (cudaStream_t)stream);
}

}  // extern "C"
