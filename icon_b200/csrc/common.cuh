// Shared helpers for libicon_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/icon_b200.h"

namespace icon {

void set_error(const char *fmt, ...);
void count_launch(int n = 1);

#define ICON_CHECK_ARG(cond, ...)                 \
    do {                                          \
        if (!(cond)) {                            \
            icon::set_error(__VA_ARGS__);         \
            return ICON_EINVAL;                   \
        }                                         \
    } while (0)

#define ICON_CUDA(expr)                                                              \
    do {                                                                             \
        cudaError_t _e = (expr);                                                     \
        if (_e != cudaSuccess) {                                                     \
            icon::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr,             \
                            cudaGetErrorString(_e));                                 \
            return ICON_ECUDA;                                                       \
        }                                                                            \
    } while (0)

// after a kernel launch
#define ICON_LAUNCHED()                 \
    do {                                \
        icon::count_launch();           \
        ICON_CUDA(cudaGetLastError());  \
    } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// cudaFuncSetAttribute is per DEVICE, the process may use several (the reference's cfg.test_gpus): remember which
// devices a kernel's opt-in has been done on.  `flags` = one static array per call site.
constexpr int ICON_MAX_DEVICES = 64;
static inline bool device_needs_setup(bool (&flags)[ICON_MAX_DEVICES], int *dev_out = nullptr) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= ICON_MAX_DEVICES) { if (dev_out) *dev_out = 0; return true; }
    if (dev_out) *dev_out = dev;
    if (flags[dev]) return false;
    flags[dev] = true;
    return true;
}
int device_sm_count();    // multiprocessors of the CURRENT device (cached per device)

// Programmatic dependent launch (PDL): the encoders are chains of ~600 short kernels; launched with the programmatic-
// stream-serialization attribute a kernel's CTAs may be scheduled while its predecessor drains, do their local set-up
// (barrier init, descriptor prefetch) and then block in pdl_wait() until the predecessor has completed
// and its writes are visible.  Every kernel launched through launch_pdl() calls pdl_launch_dependents() first thing and
// pdl_wait() before its first global-memory access; both are no-ops for a normal launch.  OFF by default (it measured
// slower than plain CUDA-graph replay: dependents park on the SMs the predecessor's tail still needs); ICON_B200_PDL=1 enables it.
bool pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                                     Args &&...args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// Normalisation statistics of one (image, channel): st[6] = {sum x, sum x^2}, each as three fp64 words that hold the
// multiples of 1, of 2^-32 and of 2^-64; zeroed by the caller.  Producers accumulate their partial sums in fp64 (x^2 of
// an fp32 x is exact there, so the variance E[x^2] - E[x]^2 keeps ~1e-16 * (mean / std)^2 relative accuracy) and add
// them here.  A partial is cut into its integer part, its fraction rounded to 2^-32 and the rest rounded to 2^-64, so
// every fp64 atomic add below is exact while the integer parts stay under 2^53 and a channel receives fewer than 2^21
// partials: the totals do not depend on the order in which blocks arrive (bitwise reproducible results, which CUDA-graph
// replay relies on).  A partial moves by at most 2^-65; the sum of a constant channel is exact, so its mean equals the
// value and the channel normalises to exactly beta.
__device__ __forceinline__ void stats_add3(double *w, double s) {
    const double a = trunc(s), r = s - a;
    const double b = rint(r * 4294967296.0) * (1.0 / 4294967296.0);
    const double c = rint((r - b) * 18446744073709551616.0) * (1.0 / 18446744073709551616.0);
    if (a != 0.0) atomicAdd(w, a);
    if (b != 0.0) atomicAdd(w + 1, b);
    if (c != 0.0) atomicAdd(w + 2, c);
}
__device__ __forceinline__ void stats_add(double *st, double s1, double s2) { stats_add3(st, s1); stats_add3(st + 3, s2); }
__device__ __forceinline__ double stats_sum(const double *st) { return st[0] + (st[1] + st[2]); }
__device__ __forceinline__ double stats_sumsq(const double *st) { return st[3] + (st[4] + st[5]); }
#endif

// carve a workspace
struct Carver {
    char *base;
    size_t off;
    explicit Carver(void *p) : base((char *)p), off(0) {}
    template <typename T>
    T *take(size_t n) {
        off = align_up(off, 256);
        T *r = (T *)(base ? base + off : nullptr);
        off += n * sizeof(T);
        return r;
    }
    size_t total() const { return align_up(off, 256); }
};

// in-place ascending heapsort of one thread's list: O(n log n) whatever its length
__device__ __forceinline__ void heap_sift(int32_t *a, int root, int n) {
    const int32_t x = a[root];
    for (int c = 2 * root + 1; c < n; c = 2 * root + 1) {
        if (c + 1 < n && a[c + 1] > a[c]) ++c;
        if (a[c] <= x) break;
        a[root] = a[c];
        root = c;
    }
    a[root] = x;
}

__device__ __forceinline__ void heap_sort_i32(int32_t *a, int n) {
    for (int i = n / 2 - 1; i >= 0; --i) heap_sift(a, i, n);
    for (int m = n - 1; m > 0; --m) {
        const int32_t t = a[0]; a[0] = a[m]; a[m] = t;
        heap_sift(a, 0, m);
    }
}

// face f's three vertex ids; false when one of them is outside [0, V)
__device__ __forceinline__ bool face_ids(const int64_t *faces, int f, int V, int id[3]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int64_t x = faces[3 * (int64_t)f + k];
        if (x < 0 || x >= V) return false;
        id[k] = (int)x;
    }
    return true;
}

// ---------------------------------------------------------------- mesh workspace layout
constexpr int TREE_MAX_LEVELS = 17;  // 4-ary implicit tree over leaves of 4 Morton-sorted faces: 4^16 leaves > 2^31 faces
constexpr int RAY_GRID = 256;        // yz cell grid for the +x ray parity
constexpr int RAY_LIST_PER_FACE = 64;

// Brick face lists for dense lattices (sdf.cu): a 32^3 grid of bricks over [-1,1]^3, one brick = 4^3 of the SDF's
// 128^3 Morton bins, so every warp of 32 Morton-adjacent lattice points lies inside one brick.  Each brick's list is
// culled from the faces of its nearby leaves, which the build gathers and sorts in shared memory.
constexpr int BRICK_AX = 32;
constexpr int NBRICK = BRICK_AX * BRICK_AX * BRICK_AX;
constexpr int BRICK_MAX_LEAVES = 4096;           // most leaves one brick's list is culled from
constexpr int BRICK_MAX_FACES = 4096;            // longest face list of one brick (it is sorted in shared memory)
constexpr int64_t BRICK_FACE_CAP = 1 << 23;      // face entries per body (48 MB of uint16 ids and float keys)
static inline int64_t brick_face_cap(int F) {
    const int64_t all = (int64_t)NBRICK * F;
    return all < BRICK_FACE_CAP ? all : BRICK_FACE_CAP;
}

struct MeshHeader {                  // device-resident, written by icon_smpl_prepare
    float y0, z0, inv_cy, inv_cz;    // ray grid origin / inverse cell size over the mesh yz box
    int ray_overflow;                // 1 -> cell lists overflowed: kernels fall back to all faces
    int brick_built;                 // 1 -> the brick lists are complete (built on the first dense call)
    int brick_overflow;              // 1 -> they did not fit: dense calls walk the tree
    int pad;
};

struct TreeBounds {                  // device-resident, written by face_tree_build
    unsigned lo[3], hi[3];           // bounding box of the faces' corners, order-preserving float encoding
    float absmax;                    // largest |coordinate| of that box (scale of the slacks of a mesh in any unit)
};

// Morton-sorted per-face records and the implicit 4-ary AABB tree over them (face_tree.cu builds it, face_tree.cuh
// walks it)
struct FaceTree {
    float4 *tri_s;        // [F][3] per-face records (a.xyz, ab.x) (ab.yz, ac.xy) (ac.z, -, -, -), sorted
    float4 *sph_s;        // [F] bounding spheres (centre xyz, radius), conservative, sorted
    int32_t *order;       // [F] sorted position -> original face id
    float4 *nodes;        // [total_nodes][2]: (min.xyz, -) (max.xyz, -), level 0 (leaves) first
    TreeBounds *bounds;
    int F;
    int nlevels;
    int lvl_cnt[TREE_MAX_LEVELS];
    int lvl_off[TREE_MAX_LEVELS];
};

struct MeshView : FaceTree {
    const float4 *tri;    // [F][3]: (a.xyz, ab.x) (ab.yz, ac.xy) (ac.z, -, -, -), original face order
    const float4 *attr;   // [F][6]: normals 9, cmap 9, vis 3, pad 3
    const float4 *rbox;   // [F][2]: (ymin, ymax, zmin, zmax) (xmax, xmin, -, -)
    float *vnormals;      // [V][3] scratch
    void *vn_ws;          // area_vertex_normals' workspace
    // ray grid
    int32_t *rcount;      // [RAY_GRID^2 + 1]
    int32_t *roff;        // [RAY_GRID^2 + 1]
    int32_t *rlist;       // [F * RAY_LIST_PER_FACE]
    MeshHeader *hdr;
    void *scan_ws;
    // brick face lists (CSR): built lazily by the first call that takes the dense path
    float4 *bxyz;         // [NBRICK] brick centres (build input)
    int32_t *bperm;       // [NBRICK] identity (build input)
    float *brec;          // [NBRICK][8] build scratch
    int32_t *bface;       // [NBRICK] original id of the face nearest the brick centre
    float *bub;           // [NBRICK] bound on the nearest distance of every point of the brick (inflated)
    int32_t *foff;        // [NBRICK + 1] face list offsets
    unsigned short *flist;   // [face_cap] sorted face positions, ascending key per list
    float *fkey;          // [face_cap] their keys: squared lower bound on the distance from any point of the brick
    int64_t face_cap;
    int V;
};
size_t mesh_ws_bytes(int V, int F);
MeshView mesh_view(const void *ws, int V, int F);
void bricks_forget(const MeshView &m);   // icon_smpl_prepare (re)fills a workspace: its brick lists are gone

// stage timing for bench.py (icon_profile_*): mark(i) records event i on `stream` when enabled
void profile_mark(int i, cudaStream_t stream);

// exclusive scan of int32 -> int64 totals; in/out may alias.  ws: scan_ws_bytes(n).
size_t scan_ws_bytes(int64_t n);
int scan_exclusive_i32(const int32_t *in, int32_t *out, int64_t n, int64_t *d_total /*may be null*/,
                       void *ws, cudaStream_t stream);

// row lists (CSR) from (owner, key) items: rows R from n items, an item with owner < 0 is dropped; off [R+1],
// list [the n' listed items], each row ascending (with ucnt: repeats dropped in place, the unique count written)
struct CsrWs {
    int32_t *cnt, *cursor;
    void *scan_ws;
};
CsrWs csr_take(Carver &c, int64_t rows);
int csr_build(const int32_t *own, const int32_t *key, int64_t n, int R, int32_t *off, int32_t *list, int32_t *ucnt,
              const CsrWs &w, cudaStream_t stream);

// per vertex, the corners 3 f + k, ascending, of every face whose three indices are in [0, V): off [V+1], list [3F]
size_t vertex_corners_ws_bytes(int V, int F);
int vertex_corners(const int64_t *faces, int F, int V, int32_t *off, int32_t *list, void *ws, cudaStream_t stream);

// pytorch3d's (pass, face) order over one vertex's corner list: passes 0, 1, 2 visit its corners 3 f + c with
// c = 1, 2, 0, each pass in ascending f; fn(f, c)
template <class Fn>
__device__ __forceinline__ void for_each_pass_corner(const int32_t *corners, int n, Fn &&fn) {
    for (int pass = 0; pass < 3; ++pass) {
        const int c = (pass + 1) % 3;
        for (int i = 0; i < n; ++i)
            if (corners[i] % 3 == c) fn(corners[i] / 3, c);
    }
}

// pytorch3d's area-weighted vertex normals (normals.cu): out [V,3]
size_t area_vertex_normals_ws_bytes(int V, int F);
int area_vertex_normals(const float *verts, int V, const int64_t *faces, int F, float *out, void *ws,
                        cudaStream_t stream);

}  // namespace icon
