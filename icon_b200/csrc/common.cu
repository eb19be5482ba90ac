// Error state, launch counter, the device-wide exclusive scan used by the compaction,
// outlier-rank and marching-cubes passes, and the row-list (CSR) builder of the mesh steps.
#include <stdarg.h>
#include <atomic>

#include <stdlib.h>

#include "common.cuh"

namespace icon {

static thread_local char g_err[512] = "";
static std::atomic<int64_t> g_launches{0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches += n; }

// ---------------------------------------------------------------- exclusive scan (int32)
// 1024 threads x 4 items = 4096 items per block; recursion on the block totals.
constexpr int SCAN_T = 1024, SCAN_I = 4, SCAN_B = SCAN_T * SCAN_I;

__global__ void __launch_bounds__(SCAN_T) k_scan_block(const int32_t *__restrict__ in,
                                                       int32_t *__restrict__ out, int64_t n,
                                                       int32_t *__restrict__ block_sums,
                                                       int64_t *__restrict__ d_total) {
    __shared__ int32_t warp_tot[32];
    int64_t base = (int64_t)blockIdx.x * SCAN_B + (int64_t)threadIdx.x * SCAN_I;
    int32_t v[SCAN_I];
    int32_t s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_I; ++i) {
        v[i] = (base + i < n) ? in[base + i] : 0;
        s += v[i];
    }
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int32_t incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        int32_t w = warp_tot[lane];
        int32_t wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int32_t t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        warp_tot[lane] = wi - w;  // exclusive warp offsets
        if (lane == 31) {
            if (block_sums) block_sums[blockIdx.x] = wi;
            if (d_total && gridDim.x == 1) *d_total = (int64_t)wi;
        }
    }
    __syncthreads();
    int32_t run = warp_tot[wid] + (incl - s);
#pragma unroll
    for (int i = 0; i < SCAN_I; ++i) {
        if (base + i < n) out[base + i] = run;
        run += v[i];
    }
}

__global__ void __launch_bounds__(SCAN_T) k_scan_add(int32_t *__restrict__ out, int64_t n,
                                                     const int32_t *__restrict__ block_offs) {
    int64_t base = (int64_t)blockIdx.x * SCAN_B + (int64_t)threadIdx.x * SCAN_I;
    int32_t o = block_offs[blockIdx.x];
#pragma unroll
    for (int i = 0; i < SCAN_I; ++i)
        if (base + i < n) out[base + i] += o;
}

size_t scan_ws_bytes(int64_t n) {
    size_t tot = 0;
    while (n > SCAN_B) {
        n = (n + SCAN_B - 1) / SCAN_B;
        tot += align_up((size_t)n * sizeof(int32_t), 256);
    }
    return tot + 256;
}

int scan_exclusive_i32(const int32_t *in, int32_t *out, int64_t n, int64_t *d_total, void *ws,
                       cudaStream_t stream) {
    if (n <= 0) {
        if (d_total) ICON_CUDA(cudaMemsetAsync(d_total, 0, sizeof(int64_t), stream));
        return ICON_OK;
    }
    int64_t nb = (n + SCAN_B - 1) / SCAN_B;
    if (nb == 1) {
        k_scan_block<<<1, SCAN_T, 0, stream>>>(in, out, n, nullptr, d_total);
        ICON_LAUNCHED();
        return ICON_OK;
    }
    int32_t *sums = (int32_t *)ws;
    void *next_ws = (char *)ws + align_up((size_t)nb * sizeof(int32_t), 256);
    k_scan_block<<<(unsigned)nb, SCAN_T, 0, stream>>>(in, out, n, sums, nullptr);
    ICON_LAUNCHED();
    int rc = scan_exclusive_i32(sums, sums, nb, d_total, next_ws, stream);
    if (rc) return rc;
    k_scan_add<<<(unsigned)nb, SCAN_T, 0, stream>>>(out, n, sums);
    ICON_LAUNCHED();
    return ICON_OK;
}

// ---------------------------------------------------------------- row lists (CSR) from (owner, key) items

__global__ void k_csr_count(const int32_t *__restrict__ own, int64_t n, int32_t *__restrict__ cnt) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && own[i] >= 0) atomicAdd(&cnt[own[i]], 1);
}

// arrival order; k_csr_sort sorts each row
__global__ void k_csr_fill(const int32_t *__restrict__ own, const int32_t *__restrict__ key, int64_t n,
                           const int32_t *__restrict__ off, int32_t *__restrict__ cursor, int32_t *__restrict__ list) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && own[i] >= 0) list[off[own[i]] + atomicAdd(&cursor[own[i]], 1)] = key[i];
}

// sort each row ascending; ucnt != NULL: drop repeats in place and write the unique count
__global__ void k_csr_sort(const int32_t *__restrict__ off, int R, int32_t *__restrict__ list,
                           int32_t *__restrict__ ucnt) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    int32_t *a = list + off[r];
    const int n = off[r + 1] - off[r];
    heap_sort_i32(a, n);
    if (!ucnt) return;
    int u = 0;
    for (int i = 0; i < n; ++i)
        if (u == 0 || a[i] != a[u - 1]) a[u++] = a[i];
    ucnt[r] = u;
}

CsrWs csr_take(Carver &c, int64_t rows) {
    CsrWs w;
    w.cnt = c.take<int32_t>((size_t)rows + 1);
    w.cursor = c.take<int32_t>((size_t)rows);
    w.scan_ws = c.take<char>(scan_ws_bytes(rows + 1));
    return w;
}

int csr_build(const int32_t *own, const int32_t *key, int64_t n, int R, int32_t *off, int32_t *list, int32_t *ucnt,
              const CsrWs &w, cudaStream_t stream) {
    ICON_CUDA(cudaMemsetAsync(w.cnt, 0, sizeof(int32_t) * ((size_t)R + 1), stream));
    ICON_CUDA(cudaMemsetAsync(w.cursor, 0, sizeof(int32_t) * (size_t)R, stream));
    const unsigned nb = (unsigned)((n + 255) / 256), rb = (unsigned)((R + 255) / 256);
    if (n > 0) {
        k_csr_count<<<nb, 256, 0, stream>>>(own, n, w.cnt);
        ICON_LAUNCHED();
    }
    int rc = scan_exclusive_i32(w.cnt, off, (int64_t)R + 1, nullptr, w.scan_ws, stream);
    if (rc) return rc;
    if (n > 0) {
        k_csr_fill<<<nb, 256, 0, stream>>>(own, key, n, off, w.cursor, list);
        ICON_LAUNCHED();
    }
    if (R > 0) {
        k_csr_sort<<<rb, 256, 0, stream>>>(off, R, list, ucnt);
        ICON_LAUNCHED();
    }
    return ICON_OK;
}

// vertex_corners items: corner i = 3 f + k under its vertex; owner -1 for every corner of a face with a bad index
__global__ void k_corner_items(const int64_t *__restrict__ faces, int F, int V, int32_t *__restrict__ own,
                               int32_t *__restrict__ key) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= F) return;
    int id[3];
    if (!face_ids(faces, f, V, id)) id[0] = id[1] = id[2] = -1;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        own[3 * f + k] = id[k];
        key[3 * f + k] = 3 * f + k;
    }
}

static size_t vc_carve(void *ws, int V, int F, int32_t **own, int32_t **key, CsrWs *csr) {
    Carver c(ws);
    int32_t *o = c.take<int32_t>(3 * (size_t)F), *k = c.take<int32_t>(3 * (size_t)F);
    const CsrWs w = csr_take(c, V);
    if (csr) *own = o, *key = k, *csr = w;
    return c.total();
}

size_t vertex_corners_ws_bytes(int V, int F) { return vc_carve(nullptr, V, F, nullptr, nullptr, nullptr); }

int vertex_corners(const int64_t *faces, int F, int V, int32_t *off, int32_t *list, void *ws, cudaStream_t stream) {
    int32_t *own, *key;
    CsrWs w;
    vc_carve(ws, V, F, &own, &key, &w);
    k_corner_items<<<(unsigned)((F + 255) / 256), 256, 0, stream>>>(faces, F, V, own, key);
    ICON_LAUNCHED();
    return csr_build(own, key, 3 * (int64_t)F, V, off, list, nullptr, w, stream);
}

static bool g_prof = false;
static cudaEvent_t g_ev[5];
static bool g_ev_ok = false;

void profile_mark(int i, cudaStream_t stream) {
    if (!g_prof) return;
    if (!g_ev_ok) {
        for (int k = 0; k < 5; ++k) cudaEventCreate(&g_ev[k]);
        g_ev_ok = true;
    }
    cudaEventRecord(g_ev[i], stream);
}

}  // namespace icon

extern "C" int icon_profile_enable(int on) {
    icon::g_prof = on != 0;
    return ICON_OK;
}
extern "C" int icon_profile_last_query(float *h_ms) {
    if (!icon::g_ev_ok) {
        icon::set_error("icon_profile_last_query: no profiled icon_query yet");
        return ICON_EINVAL;
    }
    ICON_CUDA(cudaEventSynchronize(icon::g_ev[4]));
    for (int k = 0; k < 4; ++k) ICON_CUDA(cudaEventElapsedTime(&h_ms[k], icon::g_ev[k], icon::g_ev[k + 1]));
    return ICON_OK;
}

extern "C" int icon_version(void) { return 1; }
extern "C" const char *icon_last_error(void) { return icon::g_err; }
extern "C" int64_t icon_launch_count(void) { return icon::g_launches.load(); }

namespace icon {
int device_sm_count() {
    static int counts[ICON_MAX_DEVICES] = {};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= ICON_MAX_DEVICES) return 132;
    if (!counts[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
        counts[dev] = n;
    }
    return counts[dev];
}
}  // namespace icon

namespace icon {
bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("ICON_B200_PDL");
        v = (e && e[0] == '1') ? 1 : 0;
    }
    return v == 1;
}
}  // namespace icon
