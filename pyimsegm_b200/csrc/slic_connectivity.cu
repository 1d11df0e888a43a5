// slic_connectivity.cu -- SLIC connectivity enforcement, bit-exact with oracle_enforce_connectivity().
//
// Replaces skimage.segmentation._slic._enforce_label_connectivity_cython (called from slic(),
// imsegm/superpixels.py:61-63).  The original is one sequential raster scan: every unlabelled pixel starts a
// BFS (neighbour order +x,-x,+y,-y) over same-label unlabelled pixels, truncated at max_size; a component
// smaller than min_size takes the label of the LAST already-labelled foreign neighbour the BFS looked at
// ("adjacent", 0 when none), otherwise it gets the next new label.
//
// Parallel decomposition with the same result:
//   1. 4-connected component labelling by union-find; component id = its first pixel in raster order.
//      Each 32 x 64 tile is labelled in shared memory (its local roots are the first pixels of its local components, since
//      local and global raster order agree inside a tile); only local roots take part in the global unions across the tile
//      seams, and the size and box of a component are summed from its local roots.
//   2. components >= max_size ("oversize", rare) are cut exactly as the truncated BFS would cut them: the
//      pieces depend only on the component's own shape, so one thread replays the BFS per such component.
//   3. a piece is "labelled before C" iff its first pixel precedes C's first pixel, so new labels of kept
//      pieces are a raster-order prefix count of kept roots (a popcount over a bitmap of them), and each small piece C
//      replays its own BFS to find the last foreign neighbour pixel whose piece id is < C; chains small->small are
//      followed to a kept piece (or to label 0 when the chain ends without one).
// HBM traffic: the label map read once, parent written once and read back once, out written once (16 B/px); everything else
// is per local root or per piece.
#include "common.cuh"
#include "block_scan.cuh"

namespace {

constexpr int TH = 32, TW = 64, TPIX = TH * TW; // labelling tile
constexpr int WIN = 4096;                        // small-piece window (box plus a one-pixel ring), pixels
constexpr int RANK_WORDS = 1024;                 // kept-bitmap words per rank block (32768 pixels)

// counters in ConnWs::ctr; k_small_adjacent reads its list length from [1] and its queue cursor from [2]
enum { C_OVER = 0, C_FALLBACK = 1, C_QUEUE = 2, C_LROOTS = 3, C_WINDOW = 4, C_N = 8 };

struct ConnWs {
    int* parent;    // [HW] pixel -> its tile-local root; local root -> global root after the root pass.  Flattened (pixel -> root)
                    // when oversize components or fallback pieces exist: then ~piece start on oversize pixels, VISBIT from the fallback BFS
    int* size;      // [HW] at local roots: their size, summed into the global root; at oversize piece starts: the piece size
    int* ymax;      // [HW] box at local roots, summed the same way (a root's first row is its own row)
    int* xmin;      // [HW]
    int* xmax;      // [HW]
    int* aux;       // [HW] at kept roots: new label; at small roots: -2-adjacent, or -1 when there is none
    int* lroots;    // [HW] local roots; once classified, the BFS queues of the oversize split and of the fallback
    int* window;    // [HW] small roots whose window fits WIN
    int* fallback;  // [HW] the other small roots, and small pieces of oversize splits
    int* over;      // [HW / 16 + 16] oversize roots (max_size >= 16)
    int* ctr;       // [C_N] counters, then blk and kept: one zeroed range
    int* blk;       // [n_rank_blocks] kept pieces per rank block
    unsigned* kept; // [ceil(HW / 32)] kept-piece bitmap over first pixels
};

constexpr int VISBIT = 1 << 30; // 'visited by the fallback BFS' flag kept inside parent[] (pixel indices stay below 2^30)
__device__ __forceinline__ int dec(int c) { return (c < 0 ? ~c : c) & ~VISBIT; }

// piece id of pixel p: through its local root (or, once flattened, its root) to the root, or the oversize piece it was cut into
__device__ __forceinline__ int resolve(const int* parent, int p)
{
    const int a = parent[p];
    return dec(a < 0 ? a : parent[a & ~VISBIT]);
}

__device__ __forceinline__ int find_root(const int* parent, int i)
{
    while (true) {
        int p = parent[i];
        if (p == i) return i;
        i = p;
    }
}

__device__ __forceinline__ void unite(int* parent, int a, int b)
{
    while (true) {
        a = find_root(parent, a);
        b = find_root(parent, b);
        if (a == b) return;
        if (a < b) { int t = a; a = b; b = t; }
        int old = atomicMin(&parent[a], b);
        if (old == a) return;
        a = old;
    }
}

__device__ __forceinline__ int sfind(const volatile int* par, int i)
{
    while (true) {
        int p = par[i];
        if (p == i) return i;
        i = p;
    }
}

__device__ __forceinline__ void sunite(int* par, int a, int b)
{
    while (true) {
        a = sfind(par, a);
        b = sfind(par, b);
        if (a == b) return;
        if (a < b) { int t = a; a = b; b = t; }
        int old = atomicMin(&par[a], b);
        if (old == a) return;
        a = old;
    }
}

__device__ __forceinline__ void mark_kept(int r, unsigned* kept, int* blk)
{
    atomicOr(&kept[r >> 5], 1u << (r & 31));
    atomicAdd(&blk[r / (32 * RANK_WORDS)], 1);
}

// one CTA per TH x TW tile: shared-memory union-find (smaller index wins, so a local root is the first pixel of its local
// component), parent[p] = global index of p's local root, and at each local root its size and box; local roots are listed.
__global__ void __launch_bounds__(256, 5) k_ccl_tile(const int* __restrict__ lab, int H, int W, int ntx, int* __restrict__ parent,
                                                  int* __restrict__ size, int* __restrict__ ymax, int* __restrict__ xmin,
                                                  int* __restrict__ xmax, int* __restrict__ lroots, int* ctr)
{
    constexpr int PT = TPIX / 256;
    __shared__ int s_lab[TPIX]; // labels, then local sizes
    __shared__ int s_par[TPIX];
    __shared__ int s_ymax[TPIX], s_xmin[TPIX], s_xmax[TPIX];
    __shared__ unsigned s_starts[TPIX / 32]; // run-start bits, two words per row
    const int x0 = (blockIdx.x % ntx) * TW, y0 = (blockIdx.x / ntx) * TH;
    const int tw = min(TW, W - x0), th = min(TH, H - y0);
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + 256 * k, ly = i / TW, lx = i % TW;
        s_lab[i] = (ly < th && lx < tw) ? lab[(size_t)(y0 + ly) * W + x0 + lx] : 0;
        s_ymax[i] = -1; s_xmin[i] = INT_MAX; s_xmax[i] = -1;
    }
    __syncthreads();
    // every pixel starts at the first pixel of its row run (pixels outside the image are runs of their own), so the unions
    // below only ever walk run starts
#pragma unroll
    for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + 256 * k, ly = i / TW, lx = i % TW;
        const bool start = lx == 0 || lx >= tw || ly >= th || s_lab[i - 1] != s_lab[i];
        const unsigned m = __ballot_sync(0xffffffffu, start);
        if (lane == 0) s_starts[i / 32] = m;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + 256 * k, ly = i / TW, lx = i % TW;
        const unsigned long long row = ((unsigned long long)s_starts[2 * ly + 1] << 32) | s_starts[2 * ly];
        s_par[i] = ly * TW + 63 - __clzll(row & (~0ull >> (63 - lx)));
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + 256 * k, ly = i / TW, lx = i % TW;
        if (ly == 0 || ly >= th || lx >= tw) continue;
        const int l = s_lab[i];
        if (s_lab[i - TW] != l) continue;
        if (lx > 0 && s_lab[i - 1] == l && s_lab[i - TW - 1] == l) continue; // the left pixel makes the same link
        sunite(s_par, i, i - TW);
    }
    __syncthreads();
    // run starts find their roots (compressing in place: a new parent is the root, which every reader still finds above it),
    // then every other pixel takes its run start's root
#pragma unroll
    for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + 256 * k;
        if ((s_starts[i / 32] >> (i % 32)) & 1u) s_par[i] = sfind(s_par, i);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + 256 * k;
        if (!((s_starts[i / 32] >> (i % 32)) & 1u)) s_par[i] = s_par[s_par[i]];
        s_lab[i] = 0;
    }
    __syncthreads();
    // sizes and boxes, one row run at a time: its start adds the run into the root
#pragma unroll
    for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + 256 * k, ly = i / TW, lx = i % TW;
        if (ly >= th || lx >= tw || !((s_starts[i / 32] >> (i % 32)) & 1u)) continue;
        const unsigned long long row = ((unsigned long long)s_starts[2 * ly + 1] << 32) | s_starts[2 * ly];
        const unsigned long long rest = lx == TW - 1 ? 0ull : row >> (lx + 1); // pixels past the tile's width are run starts
        const int len = rest ? __ffsll((long long)rest) : TW - lx;
        const int r = s_par[i];
        atomicAdd(&s_lab[r], len);
        atomicMax(&s_ymax[r], ly);
        atomicMin(&s_xmin[r], lx);
        atomicMax(&s_xmax[r], lx + len - 1);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + 256 * k, ly = i / TW, lx = i % TW;
        const bool valid = ly < th && lx < tw;
        const int p = (y0 + ly) * W + x0 + lx;
        const int r = s_par[i];
        const bool is_root = valid && r == i;
        if (valid) parent[p] = (y0 + r / TW) * W + x0 + r % TW;
        if (is_root) {
            size[p] = s_lab[i];
            ymax[p] = y0 + s_ymax[i]; xmin[p] = x0 + s_xmin[i]; xmax[p] = x0 + s_xmax[i];
        }
        const unsigned m = __ballot_sync(0xffffffffu, is_root);
        int base = 0;
        if (lane == 0 && m) base = atomicAdd(&ctr[C_LROOTS], __popc(m));
        base = __shfl_sync(0xffffffffu, base, 0);
        if (is_root) lroots[base + __popc(m & ((1u << lane) - 1u))] = p;
    }
}

// one thread per pair of equal labels across a tile seam: global unions of local roots
__global__ void k_ccl_seams(const int* __restrict__ lab, int H, int W, int nvs, int nhs, int* parent)
{
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nvs + nhs) return;
    int p, q;
    if (t < nvs) { // vertical seams: (y, x - 1) | (y, x)
        const int k = t / H, y = t - k * H, x = (k + 1) * TW;
        p = y * W + x; q = p - 1;
        const int l = lab[p];
        if (lab[q] != l) return;
        // inside a tile row the pair above, linked to this pair by both tiles, makes the same link
        if (y % TH != 0 && lab[p - W] == l && lab[q - W] == l) return;
    } else {       // horizontal seams: (y - 1, x) over (y, x)
        t -= nvs;
        const int k = t / W, x = t - k * W, y = (k + 1) * TH;
        p = y * W + x; q = p - W;
        const int l = lab[p];
        if (lab[q] != l) return;
        if (x % TW != 0 && lab[p - 1] == l && lab[q - 1] == l) return;
    }
    unite(parent, p, q);
}

// over the local roots: point each at its global root and add its size and box into it
__global__ void k_ccl_roots(int* parent, int* size, int* ymax, int* xmin, int* xmax, const int* __restrict__ lroots,
                            const int* __restrict__ ctr)
{
    const int n = ctr[C_LROOTS];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int lr = lroots[i];
        const int g = find_root(parent, lr);
        if (g == lr) continue;
        parent[lr] = g;
        atomicAdd(&size[g], size[lr]);
        atomicMax(&ymax[g], ymax[lr]);
        atomicMin(&xmin[g], xmin[lr]);
        atomicMax(&xmax[g], xmax[lr]);
    }
}

// over the global roots once sizes are final: oversize, kept (bitmap) or small (window or fallback list)
__global__ void k_ccl_classify(int H, int W, int min_size, int max_size, const int* __restrict__ parent, const int* __restrict__ size,
                               const int* __restrict__ ymax, const int* __restrict__ xmin, const int* __restrict__ xmax,
                               const int* __restrict__ lroots, int* ctr, int* over, int* window, int* fallback, unsigned* kept, int* blk)
{
    const int n = ctr[C_LROOTS];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int g = lroots[i];
        if (parent[g] != g) continue;
        const int s = size[g];
        if (s >= max_size) {
            over[atomicAdd(&ctr[C_OVER], 1)] = g;
        } else if (s >= min_size) {
            mark_kept(g, kept, blk);
        } else {
            const int y = g / W;
            const int wh = min(ymax[g] + 1, H - 1) - max(y - 1, 0) + 1;
            const int ww = min(xmax[g] + 1, W - 1) - max(xmin[g] - 1, 0) + 1;
            if (wh * ww <= WIN) window[atomicAdd(&ctr[C_WINDOW], 1)] = g;
            else fallback[atomicAdd(&ctr[C_FALLBACK], 1)] = g;
        }
    }
}

// parent[p] = root of p in place (roots keep their value), for the oversize split and the fallback BFS, which read one hop;
// a no-op when neither has work
__global__ void k_ccl_flatten(int n, int* parent, const int* __restrict__ ctr)
{
    if (ctr[C_OVER] == 0 && ctr[C_FALLBACK] == 0) return;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) parent[p] = parent[parent[p]];
}

// one thread per oversize component: replay the truncated BFS over its box; assigned pixels get comp = ~piece_root, and each
// piece is kept or listed for the fallback BFS
__global__ void k_oversize_split(int H, int W, int* comp, int* size, const int* __restrict__ ymax, const int* __restrict__ xmin,
                                 const int* __restrict__ xmax, int min_size, int max_size, const int* __restrict__ list, int* ctr,
                                 int* fallback, unsigned* kept, int* blk, int* queue)
{
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ctr[C_OVER]) return;
    const int C = list[i];
    const int4 bb = make_int4(C / W, ymax[C], xmin[C], xmax[C]);
    int* q = queue + (size_t)i * max_size;
    const int total = size[C];
    int assigned = 0;
    for (int y = bb.x; y <= bb.y && assigned < total; ++y)
        for (int x = bb.z; x <= bb.w && assigned < total; ++x) {
            int p = y * W + x;
            if (comp[p] != C) continue; // foreign, or already assigned (negative)
            int start = p;
            comp[p] = ~start;
            q[0] = p;
            int n = 1, v = 0;
            while (v < n && n < max_size) {
                int cp = q[v];
                int cy = cp / W, cx = cp - cy * W;
                const int nx[4] = { cx + 1, cx - 1, cx, cx };
                const int ny[4] = { cy, cy, cy + 1, cy - 1 };
                for (int d = 0; d < 4; ++d) {
                    if (nx[d] < 0 || nx[d] >= W || ny[d] < 0 || ny[d] >= H) continue;
                    int np_ = ny[d] * W + nx[d];
                    if (comp[np_] == C) {
                        comp[np_] = ~start;
                        q[n++] = np_;
                        if (n >= max_size) break;
                    }
                }
                ++v;
            }
            size[start] = n;
            assigned += n;
            if (n >= min_size) mark_kept(start, kept, blk);
            else fallback[atomicAdd(&ctr[C_FALLBACK], 1)] = start;
        }
}

// one CTA per RANK_WORDS words of the kept bitmap: a kept piece's label is the number of kept first pixels before it
__global__ void __launch_bounds__(256) k_kept_ranks(int n_words, const unsigned* __restrict__ kept, const int* __restrict__ blk,
                                                    int* aux, int* n_labels_out)
{
    constexpr int WPT = RANK_WORDS / 256;
    int part = 0;
    for (int j = threadIdx.x; j < (int)blockIdx.x; j += 256) part += blk[j];
    unsigned bits[WPT];
    int c = 0;
#pragma unroll
    for (int k = 0; k < WPT; ++k) {
        const int w = blockIdx.x * RANK_WORDS + threadIdx.x * WPT + k;
        bits[k] = w < n_words ? kept[w] : 0u;
        c += __popc(bits[k]);
    }
    // base = the kept first pixels of the rank blocks before this one, then the exclusive block scan of c
    int base, tot;
    cta_exclusive_sum<256>(part, base);
    int label = base + cta_exclusive_sum<256>(c, tot);
#pragma unroll
    for (int k = 0; k < WPT; ++k) {
        const int w = blockIdx.x * RANK_WORDS + threadIdx.x * WPT + k;
        for (unsigned b = bits[k]; b; b &= b - 1) aux[w * 32 + __ffs(b) - 1] = label++;
    }
    // when no component reaches min_size everything is merged into label 0: the map still holds one label
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *n_labels_out = base + tot > 0 ? base + tot : 1;
}

// one CTA per small piece whose box plus a one-pixel ring fits WIN pixels: the window's piece ids go to shared memory and one
// thread replays the piece's BFS there, remembering the last foreign earlier-labelled neighbour piece.  A window piece is a
// whole component below max_size, so its BFS is never truncated.
__global__ void __launch_bounds__(256) k_small_window(int H, int W, const int* __restrict__ parent, const int* __restrict__ ymax,
                                                      const int* __restrict__ xmin, const int* __restrict__ xmax,
                                                      const int* __restrict__ list, const int* __restrict__ ctr, int* __restrict__ aux)
{
    __shared__ int s_id[WIN];
    __shared__ int s_q[WIN]; // queue entries (window row << 16) | window column
    const int n_small = ctr[C_WINDOW];
    for (int i = blockIdx.x; i < n_small; i += gridDim.x) {
        const int C = list[i];
        const int y = C / W, x = C - y * W;
        const int wy0 = max(y - 1, 0), wx0 = max(xmin[C] - 1, 0);
        const int wh = min(ymax[C] + 1, H - 1) - wy0 + 1, ww = min(xmax[C] + 1, W - 1) - wx0 + 1;
        const int area = wh * ww;
#pragma unroll 4
        for (int j = threadIdx.x; j < area; j += 256) {
            const int jy = j / ww;
            s_id[j] = resolve(parent, (wy0 + jy) * W + wx0 + j - jy * ww);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int adjacent = -1;
            const int cy0 = y - wy0, cx0 = x - wx0;
            s_q[0] = (cy0 << 16) | cx0;
            s_id[cy0 * ww + cx0] = INT_MAX; // visited: neither C nor below C
            int n = 1;
            for (int v = 0; v < n; ++v) {
                const int cy = s_q[v] >> 16, cx = s_q[v] & 0xffff;
                const int c = cy * ww + cx, gy = wy0 + cy, gx = wx0 + cx;
                // the four neighbours in the original's order (+x, -x, +y, -y); an in-image neighbour lies inside the window
                const bool ok4[4] = { gx + 1 < W, gx > 0, gy + 1 < H, gy > 0 };
                const int nc4[4] = { c + 1, c - 1, c + ww, c - ww };
                const int nq4[4] = { (cy << 16) | (cx + 1), (cy << 16) | (cx - 1), ((cy + 1) << 16) | cx, ((cy - 1) << 16) | cx };
                int r4[4];
#pragma unroll
                for (int d = 0; d < 4; ++d) r4[d] = ok4[d] ? s_id[nc4[d]] : INT_MAX;
#pragma unroll
                for (int d = 0; d < 4; ++d) {
                    if (r4[d] == C) { // the four neighbours of one pixel are distinct
                        s_id[nc4[d]] = INT_MAX;
                        s_q[n++] = nq4[d];
                    } else if (r4[d] < C) {
                        adjacent = r4[d];
                    }
                }
            }
            aux[C] = adjacent >= 0 ? -2 - adjacent : -1; // small roots store -2-adjacent (kept roots store label >= 0)
        }
        __syncthreads();
    }
}

// one thread per small piece the window does not take: replay its BFS, remember the last foreign earlier-labelled neighbour piece.
// The kernel is a chain of dependent loads per piece (queue entry -> four neighbours), as long as the largest small piece: the queue of
// a piece (fewer than min_size entries) lives in SHARED memory when it fits (SQ: 32 threads per CTA, entry j of lane l at q[32 j + l]),
// which takes one of the two global round trips out of every BFS step.
template <bool SQ>
__global__ void __launch_bounds__(SQ ? 32 : 256) k_small_adjacent(int H, int W, int* comp, const int* __restrict__ size, int max_size,
                                                                   const int* __restrict__ list, int* ctr, int* aux, int* queue)
{
    extern __shared__ int s_q[];
    const int n_small = ctr[1];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_small; i += gridDim.x * blockDim.x) {
        const int C = list[i];
        int* q = SQ ? s_q + threadIdx.x : queue + atomicAdd(&ctr[2], size[C]);
        constexpr int QS = SQ ? 32 : 1;
        int adjacent = -1;
        q[0] = C;
        // the visited flag lives in comp[] itself (only this thread writes the pixels of its own piece; every reader masks the
        // flag with dec()), so one round of four independent loads per BFS step is all the memory latency there is
        comp[C] = (comp[C] < 0 ? ~(dec(comp[C]) | VISBIT) : (comp[C] | VISBIT));
        int n = 1, v = 0;
        while (v < n && n < max_size) {
            const int cp = q[v * QS];
            const int cy = cp / W, cx = cp - cy * W;
            // the four neighbours in the original's order (+x, -x, +y, -y)
            const int np4[4] = { cx + 1 < W ? cp + 1 : -1, cx > 0 ? cp - 1 : -1, cy + 1 < H ? cp + W : -1, cy > 0 ? cp - W : -1 };
            int raw4[4];
#pragma unroll
            for (int d = 0; d < 4; ++d) raw4[d] = np4[d] >= 0 ? comp[np4[d]] : 0;
#pragma unroll
            for (int d = 0; d < 4; ++d) {
                if (np4[d] < 0) continue;
                const int raw = raw4[d];
                const int r = dec(raw);
                if (r == C) {
                    const bool seen = ((raw < 0 ? ~raw : raw) & VISBIT) != 0; // the four neighbours of one pixel are distinct
                    if (!seen) {
                        comp[np4[d]] = raw < 0 ? ~((~raw) | VISBIT) : (raw | VISBIT);
                        q[(n++) * QS] = np4[d];
                        if (n >= max_size) break;
                    }
                } else if (r < C) {
                    adjacent = r;
                }
            }
            ++v;
        }
        aux[C] = adjacent >= 0 ? -2 - adjacent : -1; // small roots store -2-adjacent (kept roots store label >= 0)
    }
}

// WRITE_PX pixels per thread, a block width apart: their three dependent loads (parent, the local root's parent, aux) overlap
constexpr int WRITE_PX = 4;
__global__ void __launch_bounds__(256) k_ccl_write(int n, const int* __restrict__ parent, const int* __restrict__ aux,
                                                   int* __restrict__ out)
{
    const int p0 = blockIdx.x * 256 * WRITE_PX + threadIdx.x;
    int r[WRITE_PX], a[WRITE_PX];
#pragma unroll
    for (int k = 0; k < WRITE_PX; ++k) r[k] = p0 + 256 * k < n ? parent[p0 + 256 * k] : 0;
#pragma unroll
    for (int k = 0; k < WRITE_PX; ++k) r[k] = dec(r[k] < 0 ? r[k] : parent[r[k] & ~VISBIT]);
#pragma unroll
    for (int k = 0; k < WRITE_PX; ++k) a[k] = aux[r[k]];
#pragma unroll
    for (int k = 0; k < WRITE_PX; ++k) {
        // follow small -> adjacent chains (each hop goes to a piece with a smaller root index)
        while (a[k] < -1) { r[k] = -2 - a[k]; a[k] = aux[r[k]]; }
        if (p0 + 256 * k < n) out[p0 + 256 * k] = a[k] < 0 ? 0 : a[k];
    }
}

static size_t carve(ConnWs& w, void* ws, size_t bytes, int H, int W, int* n_zero)
{
    WsCarver c(ws, bytes);
    size_t n = (size_t)H * W;
    w.parent = c.take<int>(n); w.size = c.take<int>(n);
    w.ymax = c.take<int>(n); w.xmin = c.take<int>(n); w.xmax = c.take<int>(n);
    w.aux = c.take<int>(n); w.lroots = c.take<int>(n); w.window = c.take<int>(n); w.fallback = c.take<int>(n);
    w.over = c.take<int>(n / 16 + 16);
    const size_t n_words = (n + 31) / 32, n_blk = (n_words + RANK_WORDS - 1) / RANK_WORDS;
    w.ctr = c.take<int>(C_N + n_blk + n_words);
    w.blk = w.ctr + C_N;
    w.kept = (unsigned*)(w.blk + n_blk);
    *n_zero = (int)(C_N + n_blk + n_words);
    return isb_align(c.off);
}

} // namespace

extern "C" size_t isb_connectivity_workspace_bytes(int H, int W)
{
    ConnWs w;
    int n_zero;
    return carve(w, nullptr, 0, H, W, &n_zero);
}

extern "C" int isb_enforce_connectivity(const int32_t* labels, int H, int W, int min_size, int max_size, int32_t* out,
                                        int32_t* n_labels_out, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(labels && out && n_labels_out && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && (long long)H * W < (1LL << 30), "bad image size (at most 2^30 pixels)");
    if (max_size < 1) max_size = 1;
    ISB_REQUIRE(max_size >= 16, "max_size < 16 is not supported on the device path (oversize table bound)");
    ConnWs w;
    int n_zero;
    size_t need = carve(w, ws, ws_bytes, H, W, &n_zero);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_CONN, st);
    const int n = H * W;
    const int ntx = (W + TW - 1) / TW, nty = (H + TH - 1) / TH;
    const int n_words = (n + 31) / 32, n_rank = (n_words + RANK_WORDS - 1) / RANK_WORDS;
    int dev = 0, sms = 0;
    ISB_CUDA_CHECK(cudaGetDevice(&dev));
    ISB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.ctr, 0, sizeof(int) * (size_t)n_zero, st));
    k_ccl_tile<<<ntx * nty, 256, 0, st>>>(labels, H, W, ntx, w.parent, w.size, w.ymax, w.xmin, w.xmax, w.lroots, w.ctr);
    ISB_LAUNCH_CHECK();
    const int nvs = (ntx - 1) * H, nhs = (nty - 1) * W;
    if (nvs + nhs > 0) {
        k_ccl_seams<<<(nvs + nhs + 255) / 256, 256, 0, st>>>(labels, H, W, nvs, nhs, w.parent);
        ISB_LAUNCH_CHECK();
    }
    k_ccl_roots<<<sms * 4, 256, 0, st>>>(w.parent, w.size, w.ymax, w.xmin, w.xmax, w.lroots, w.ctr);
    ISB_LAUNCH_CHECK();
    k_ccl_classify<<<sms * 4, 256, 0, st>>>(H, W, min_size, max_size, w.parent, w.size, w.ymax, w.xmin, w.xmax, w.lroots, w.ctr,
                                            w.over, w.window, w.fallback, w.kept, w.blk);
    ISB_LAUNCH_CHECK();
    k_ccl_flatten<<<sms * 8, 256, 0, st>>>(n, w.parent, w.ctr);
    ISB_LAUNCH_CHECK();
    // the local-root list is dead once classified: it becomes the BFS queue space
    const int n_over_max = n / max_size + 1;
    k_oversize_split<<<(n_over_max + 63) / 64, 64, 0, st>>>(H, W, w.parent, w.size, w.ymax, w.xmin, w.xmax, min_size, max_size, w.over,
                                                            w.ctr, w.fallback, w.kept, w.blk, w.lroots);
    ISB_LAUNCH_CHECK();
    k_kept_ranks<<<n_rank, 256, 0, st>>>(n_words, w.kept, w.blk, w.aux, n_labels_out);
    ISB_LAUNCH_CHECK();
    k_small_window<<<sms * 6, 256, 0, st>>>(H, W, w.parent, w.ymax, w.xmin, w.xmax, w.window, w.ctr, w.aux);
    ISB_LAUNCH_CHECK();
    // the fallback reads the real count of its pieces and strides over them
    if (min_size >= 1 && min_size <= 512) {
        // a small piece has fewer than min_size pixels: its queue fits min_size entries of shared memory per thread
        const size_t smem = sizeof(int) * 32 * (size_t)min_size;
        ISB_CUDA_CHECK(cudaFuncSetAttribute(k_small_adjacent<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_small_adjacent<true><<<sms * 16, 32, smem, st>>>(H, W, w.parent, w.size, max_size, w.fallback, w.ctr, w.aux, w.lroots);
    } else {
        k_small_adjacent<false><<<sms * 8, 256, 0, st>>>(H, W, w.parent, w.size, max_size, w.fallback, w.ctr, w.aux, w.lroots);
    }
    ISB_LAUNCH_CHECK();
    k_ccl_write<<<(n + 256 * WRITE_PX - 1) / (256 * WRITE_PX), 256, 0, st>>>(n, w.parent, w.aux, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
