// psm_speckle.cuh -- speckle removal on the disparity maps (psm_set_speckle_filter): OpenCV's
// cv::filterSpeckles(map, newVal = 0, maxSpeckleSize, maxDiff) on both views.
//
// Definition (independent of any visiting order): pixels of value 0 belong to no blob; two 4-neighbours p, q, both
// non-zero, are in the same blob when |m(p) - m(q)| <= max_diff (as int); every pixel of a blob of at most max_size
// pixels becomes 0, every other pixel keeps its value.
//
// GPU mapping: block-based union-find connected-component labelling over a label plane of int32 (the global index of a
// pixel's parent; a root points at itself) and a count plane of int32, both W x H per view.  Every kernel takes both
// views (blockIdx.z = view).  Labels only ever decrease, so lab[x] <= x at all times and a root is the smallest index
// of its tree.
//   1. speckle_local_kernel: one kSpTile x kSpTile tile per CTA, labelled in shared memory: each row's runs of joined
//      pixels by a warp ballot, then an atomicMin union-find over the runs of neighbouring rows; each pixel's label is
//      the global index of its tile root.  Zeroes the count plane.
//   2. speckle_seam_kernel: one thread per edge across a tile border, united with the lock-free atomicMin union on the
//      global label plane (no path compression while unions run), unless the previous edge along the seam already
//      implies it.
//   3. speckle_count_kernel: the root of every non-zero pixel, with full path compression (every write is the final
//      root, so concurrent compressions agree); the pixel's label becomes its root.  One atomicAdd per distinct root
//      per warp (__match_any_sync), so a map-wide blob adds once per warp, not once per pixel.
//   4. speckle_paint_kernel: out = (m != 0 && count[root] <= max_size) ? 0 : m.
// The result depends only on the partition into blobs, not on which labels the races produce.
#pragma once
#include "psm_common.cuh"

namespace psm {

constexpr int kSpTile = 32;                  // tile side: 1024 pixels per CTA
constexpr int kSpRows = 8;                   // threads per tile column: kSpTile / kSpRows rows per thread
constexpr int kSpThreads = kSpTile * kSpRows;
constexpr int kSpSeamThreads = 256;
static_assert(kSpTile == 32, "a tile row is one warp (the run ballot and the count kernel's __match_any_sync)");

// both views' maps, labels and counts of one launch; view v's planes start at v * npix
template <typename T>
struct SpeckleArgs {
    const T* map[2];
    int* lab;
    int* cnt;
    int W, H;
    int max_diff;
    // view v's map (selected, not indexed: an indexed parameter array would go through a local-memory copy)
    __device__ __forceinline__ const T* view_map(int v) const { return v ? map[1] : map[0]; }
};

__device__ __forceinline__ bool sp_joined(int a, int b, int max_diff)
{
    return a != 0 && b != 0 && abs(a - b) <= max_diff;
}

// the root of x, reading parents past L1 (other threads link and compress them)
__device__ __forceinline__ int sp_find(const int* lab, int x)
{
    int p = __ldcg(lab + x);
    while (p != x) { x = p; p = __ldcg(lab + x); }
    return x;
}

// the lock-free union of a's and b's trees: link the larger root under the smaller with atomicMin; when the target was
// no longer a root (another thread linked it first), continue from the parent the atomic returned
__device__ __forceinline__ void sp_unite(int* lab, int a, int b)
{
    for (;;) {
        a = sp_find(lab, a);
        b = sp_find(lab, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(lab + a, b);
        if (old == a) return;
        a = old;
    }
}

// shared-memory twin of sp_find / sp_unite for the tile labels (local indices)
__device__ __forceinline__ int sp_find_local(const volatile int* s, int x)
{
    int p = s[x];
    while (p != x) { x = p; p = s[x]; }
    return x;
}

__device__ __forceinline__ void sp_unite_local(int* s, int a, int b)
{
    for (;;) {
        a = sp_find_local(s, a);
        b = sp_find_local(s, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }
        const int old = atomicMin(s + a, b);
        if (old == a) return;
        a = old;
    }
}

// one warp per tile row (blockDim = (kSpTile, kSpRows)): each row's runs of joined pixels are labelled with a ballot, so
// the shared-memory union-find only unites runs of neighbouring rows
template <typename T>
__global__ void __launch_bounds__(kSpThreads) speckle_local_kernel(SpeckleArgs<T> a)
{
    __shared__ int s_lab[kSpTile * kSpTile];
    __shared__ int s_val[kSpTile * kSpTile];
    const int v = blockIdx.z;
    const size_t npix = (size_t)a.W * a.H;
    const T* m = a.view_map(v);
    int* lab = a.lab + v * npix;
    int* cnt = a.cnt + v * npix;
    const int tx = threadIdx.x, x = blockIdx.x * kSpTile + tx;
    const int y0 = blockIdx.y * kSpTile;
#pragma unroll
    for (int k = 0; k < kSpTile / kSpRows; ++k) {
        const int ty = threadIdx.y + k * kSpRows, y = y0 + ty;
        s_val[ty * kSpTile + tx] = x < a.W && y < a.H ? (int)m[(size_t)y * a.W + x] : 0;   // outside the map: 0
    }
    __syncthreads();
    // runs: a pixel joined to its left neighbour takes the label of the first pixel of its run
#pragma unroll
    for (int k = 0; k < kSpTile / kSpRows; ++k) {
        const int ty = threadIdx.y + k * kSpRows, i = ty * kSpTile + tx;
        const bool cont = tx > 0 && sp_joined(s_val[i - 1], s_val[i], a.max_diff);
        const unsigned starts = __ballot_sync(0xffffffffu, !cont);
        s_lab[i] = ty * kSpTile + 31 - __clz(starts & (0xffffffffu >> (31 - tx)));
    }
    __syncthreads();
    // rows: unite each pixel with the one below, unless the pair to the left (joined to both) already connects them
#pragma unroll
    for (int k = 0; k < kSpTile / kSpRows; ++k) {
        const int ty = threadIdx.y + k * kSpRows, i = ty * kSpTile + tx;
        if (ty + 1 == kSpTile) continue;
        const int c = s_val[i], b = s_val[i + kSpTile];
        if (!sp_joined(c, b, a.max_diff)) continue;
        if (tx > 0) {
            const int cl = s_val[i - 1], bl = s_val[i + kSpTile - 1];
            if (sp_joined(cl, bl, a.max_diff) && sp_joined(cl, c, a.max_diff) && sp_joined(bl, b, a.max_diff)) continue;
        }
        sp_unite_local(s_lab, i, i + kSpTile);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kSpTile / kSpRows; ++k) {
        const int ty = threadIdx.y + k * kSpRows, y = y0 + ty, i = ty * kSpTile + tx;
        if (x < a.W && y < a.H) {
            const int r = sp_find_local(s_lab, i);
            const size_t g = (size_t)y * a.W + x;
            lab[g] = (int)((size_t)(y0 + r / kSpTile) * a.W + blockIdx.x * kSpTile + r % kSpTile);
            cnt[g] = 0;
        }
    }
}

// thread t < nv: the edge across vertical seam t / H at row t % H; then one thread per edge across horizontal seams
template <typename T>
__global__ void __launch_bounds__(kSpSeamThreads) speckle_seam_kernel(SpeckleArgs<T> a, int nv, int nh)
{
    const int v = blockIdx.z;
    const size_t npix = (size_t)a.W * a.H;
    const T* m = a.view_map(v);
    int* lab = a.lab + v * npix;
    const long t = (long)blockIdx.x * kSpSeamThreads + threadIdx.x;
    int p, q, along;   // the edge p - q and the step to the previous edge along its seam (0: none to rely on)
    if (t < nv) {
        const int x = (int)(t / a.H + 1) * kSpTile, y = (int)(t % a.H);
        p = y * a.W + x - 1;
        q = p + 1;
        along = y % kSpTile ? a.W : 0;
    } else if (t < (long)nv + nh) {
        const long u = t - nv;
        const int y = (int)(u / a.W + 1) * kSpTile, x = (int)(u % a.W);
        q = y * a.W + x;
        p = q - a.W;
        along = x % kSpTile ? 1 : 0;
    } else {
        return;
    }
    const int mp = m[p], mq = m[q];
    if (!sp_joined(mp, mq, a.max_diff)) return;
    // The previous edge p' - q' along the seam, with p' - p and q' - q joined, already connects p and q.  Only inside a
    // tile's side: there p' - p and q' - q are tile edges the local kernel united, and p' - q' is united here or rests on
    // the edge before it in turn, back to the side's first edge, which is always united.  (Across a corner both seams'
    // edges would rest on each other.)  On smooth blobs this leaves one union per run of joined edges per tile side.
    if (along) {
        const int mp2 = m[p - along], mq2 = m[q - along];
        if (sp_joined(mp2, mq2, a.max_diff) && sp_joined(mp2, mp, a.max_diff) && sp_joined(mq2, mq, a.max_diff)) return;
    }
    sp_unite(lab, p, q);
}

template <typename T>
__global__ void __launch_bounds__(kSpThreads) speckle_count_kernel(SpeckleArgs<T> a)
{
    const int v = blockIdx.z;
    const size_t npix = (size_t)a.W * a.H;
    const T* m = a.view_map(v);
    int* lab = a.lab + v * npix;
    int* cnt = a.cnt + v * npix;
    const int x = blockIdx.x * kSpTile + threadIdx.x, y = blockIdx.y * kSpRows + threadIdx.y;
    const int lane = threadIdx.x;   // a warp is one row of kSpTile = 32 pixels
    const size_t g = (size_t)y * a.W + x;
    const bool valid = x < a.W && y < a.H && m[g] != 0;
    const unsigned act = __ballot_sync(0xffffffffu, valid);
    if (!valid) return;
    // pixels of one tile share their label: the first lane of each label walks the tree for all of them
    const int l = lab[g];
    const unsigned same = __match_any_sync(act, l);
    const int lead = __ffs(same) - 1;
    int r = 0;
    if (lane == lead) {
        r = sp_find(lab, l);
        for (int n = l; n != r;) {   // full compression of the walked path
            const int p = __ldcg(lab + n);
            lab[n] = r;
            n = p;
        }
    }
    r = __shfl_sync(act, r, lead);
    if (r != l) lab[g] = r;
    const unsigned peers = __match_any_sync(act, r);
    if (lane == __ffs(peers) - 1) atomicAdd(cnt + r, __popc(peers));
}

template <typename T>
__global__ void __launch_bounds__(kSpThreads) speckle_paint_kernel(SpeckleArgs<T> a, int max_size, T* out_l, T* out_r)
{
    const int v = blockIdx.z;
    const size_t npix = (size_t)a.W * a.H;
    const int x = blockIdx.x * kSpTile + threadIdx.x, y = blockIdx.y * kSpRows + threadIdx.y;
    if (x >= a.W || y >= a.H) return;
    const size_t g = (size_t)y * a.W + x;
    const T d = a.view_map(v)[g];
    T* out = v ? out_r : out_l;
    out[g] = d != 0 && a.cnt[v * npix + a.lab[v * npix + g]] <= max_size ? T(0) : d;
}

}  // namespace psm
