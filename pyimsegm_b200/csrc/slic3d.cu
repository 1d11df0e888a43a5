// slic3d.cu -- SLIC superpixels of a single-channel VOLUME, bit-exact with oracle/slic3d_oracle.c.
//
// Replaces skimage.segmentation.slic(vol, n_segments, compactness, multichannel=False, spacing=space, sigma=1) as called from
// imsegm/superpixels.py:104-106 (segment_slic_img3d_gray) -- the first stage of pipe_gray3d_slic_features_model_graphcut
// (imsegm/pipelines.py:382-431).  Same decomposition as the 2-D path (slic_prepare.cu / slic_kmeans.cu / slic_connectivity.cu),
// written for generality rather than speed: the reference's volumes are small (100 x 100 x 10, 5 x 125 x 150 in its doctests).
//
//  * pre-blur: scipy gaussian_filter, one symmetric 1-D correlate per axis (z, y, x), sigma / spacing per axis
//  * assignment: the original takes, per voxel, the minimum over the clusters whose +-2*step window holds it of (distance,
//    index) in lexicographic order.  Cluster-centric here in two passes: atomicMin of the distance bit pattern (non-negative
//    doubles order like their bits), then atomicMin of the cluster index among the clusters that reach that minimum.
//  * centroid update: raster-order sequential double sum of the values (one warp per cluster walks the box of its members,
//    ballots and compacts the members of a 32-voxel chunk, lane 0 adds them one by one); coordinate sums are integers.
//  * connectivity: union-find components (root = first raster voxel), components >= max_size cut by replaying the truncated BFS
//    (one thread per such component), pieces < min_size replay their own BFS to find the last earlier-labelled neighbour piece,
//    chains of small pieces are followed to a kept piece; new labels = raster-order rank of the kept pieces.
//  * slab mode (isb_slic3d_slab_*): the same sweeps over one z-slab of a volume per GPU; the scan clips each window to the slab's
//    slices, the owner of a cluster's centre slice writes its sums to an int64 exchange record (k3_update), k3_import takes the
//    records merged over the slabs.
// All distances in IEEE double without FMA, in the oracle's operation order.
#include "common.cuh"
#include "block_scan.cuh"
#include <float.h>
#include <limits.h>

namespace {

// dtype -> f64 with skimage's img_as_float scale (1/255, 1/65535 for the integer types; floats unchanged)
__global__ void k3_load(const void* __restrict__ vol, int dtype, size_t n, double* __restrict__ out)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double v = load_as_f64(vol, dtype, i);
    if (dtype == ISB_U8) v = __ddiv_rn(v, 255.0);
    else if (dtype == ISB_U16) v = __ddiv_rn(v, 65535.0);
    out[i] = v;
}

// the array holds slices [z_off, z_off + S) of a volume of depth D: z reflects at the volume's borders, so a slice whose window
// of +- r_z slices lies inside the array (clipped to the volume) gets the value the whole volume gives it
__global__ void k3_blur_axis(const double* __restrict__ in, double* __restrict__ out, int S, int H, int W, int z_off, int D, int axis,
                             const double* __restrict__ w, int r)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)S * H * W) return;
    const int x = (int)(i % W), y = (int)((i / W) % H), z = (int)(i / ((size_t)H * W)) + z_off;
    const int c = axis == 0 ? z : (axis == 1 ? y : x), n = axis == 0 ? D : (axis == 1 ? H : W);
    const long st = axis == 0 ? (long)H * W : (axis == 1 ? W : 1);
    // the slices within r_z of a slab's ends read past the array: those are clamped to it, and their values are not used
    const int lo = axis == 0 ? z_off : 0, hi = axis == 0 ? z_off + S - 1 : n - 1;
    double t = __dmul_rn(in[i], w[0]);
    for (int j = r; j >= 1; --j) {
        const double a = in[i + (long)(min(max(reflect_index(c - j, n), lo), hi) - c) * st];
        const double b = in[i + (long)(min(max(reflect_index(c + j, n), lo), hi) - c) * st];
        t = __dadd_rn(t, __dmul_rn(__dadd_rn(a, b), w[j]));
    }
    out[i] = t;
}

__global__ void k3_scale(const double* __restrict__ in, double* __restrict__ out, size_t n, double ratio)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = __dmul_rn(in[i], ratio);
}

struct Km3 {
    double* cz; double* cy; double* cx; double* cv;   // [n]
    int* alive;                                        // [n]
    int* bb;                                           // [n][6] member box zmin, zmax, ymin, ymax, xmin, xmax
    unsigned long long* dist;                          // [V] bit pattern of the current minimum
    int* lab_new;                                      // [V]
    int n, D, H, W, step_z, step_y, step_x;
    int z_off, Dg;                                     // voxel memory: slices [z_off, z_off + D) of a volume of depth Dg
    int own_lo, own_hi, halo;                          // slab mode (xchg != null in k3_update): the owned slices and the halo
    double sz, sy, sx, sw;
};

__device__ __forceinline__ void window3(double c, int step, int size, int& lo_i, int& hi_i)
{
    double lo = __dsub_rn(c, (double)(2 * step)); if (0.0 > lo) lo = 0.0;
    double hi = __dadd_rn(__dadd_rn(c, (double)(2 * step)), 1.0); if ((double)size < hi) hi = (double)size;
    lo_i = (int)lo; hi_i = (int)hi;
}

__global__ void k3_seed(Km3 s, const double* __restrict__ seeds)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= s.n) return;
    s.cz[k] = seeds[3 * k]; s.cy[k] = seeds[3 * k + 1]; s.cx[k] = seeds[3 * k + 2]; s.cv[k] = 0.0;
    s.alive[k] = 1;
}

__global__ void k3_clear(Km3 s)
{
    const size_t V = (size_t)s.D * s.H * s.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < V) { s.dist[i] = 0x7FEFFFFFFFFFFFFFull; s.lab_new[i] = INT_MAX; }   // DBL_MAX
    if (i < (size_t)s.n) {
        int* b = s.bb + 6 * i;
        b[0] = INT_MAX; b[1] = -1; b[2] = INT_MAX; b[3] = -1; b[4] = INT_MAX; b[5] = -1;
    }
}

// PASS 0: dist[v] = min over clusters of the distance;  PASS 1: lab_new[v] = lowest cluster index that reaches it
template <int PASS>
__global__ void __launch_bounds__(256) k3_scan(Km3 s, const double* __restrict__ vol)
{
    const int k = blockIdx.x;
    if (!s.alive[k]) return;
    const double cz = s.cz[k], cy = s.cy[k], cx = s.cx[k], cv = s.cv[k];
    int z0, z1, y0, y1, x0, x1;
    window3(cz, s.step_z, s.Dg, z0, z1);
    window3(cy, s.step_y, s.H, y0, y1);
    window3(cx, s.step_x, s.W, x0, x1);
    z0 = max(z0, s.z_off); z1 = min(z1, s.z_off + s.D);      // the slices this slab holds (all of them for a whole volume)
    if (z1 <= z0) return;
    const int wy = y1 - y0, wx = x1 - x0;
    const long total = (long)(z1 - z0) * wy * wx;
    for (long i = threadIdx.x; i < total; i += blockDim.x) {
        const int x = x0 + (int)(i % wx), y = y0 + (int)((i / wx) % wy), z = z0 + (int)(i / ((long)wx * wy));
        const double tz = __dmul_rn(s.sz, __dsub_rn(cz, (double)z));
        const double ty = __dmul_rn(s.sy, __dsub_rn(cy, (double)y));
        const double tx = __dmul_rn(s.sx, __dsub_rn(cx, (double)x));
        double dc = __dmul_rn(__dadd_rn(__dadd_rn(__dmul_rn(tz, tz), __dmul_rn(ty, ty)), __dmul_rn(tx, tx)), s.sw);
        const size_t p = ((size_t)(z - s.z_off) * s.H + y) * s.W + x;
        const double d0 = __dsub_rn(vol[p], cv);
        dc = __dadd_rn(dc, __dmul_rn(d0, d0));
        const unsigned long long bits = (unsigned long long)__double_as_longlong(dc);
        if (PASS == 0) { if (bits < 0x7FEFFFFFFFFFFFFFull) atomicMin(&s.dist[p], bits); }   // 'dist > d' from DBL_MAX: strict
        else if (bits == s.dist[p]) atomicMin(&s.lab_new[p], k);
    }
}

// take the new labels (a voxel no window reached keeps its label) and grow the member boxes
__global__ void k3_commit(Km3 s, int* __restrict__ labels)
{
    const size_t V = (size_t)s.D * s.H * s.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    int l = s.lab_new[i];
    if (l != INT_MAX) labels[i] = l; else l = labels[i];
    const int x = (int)(i % s.W), y = (int)((i / s.W) % s.H), z = (int)(i / ((size_t)s.H * s.W)) + s.z_off;
    int* b = s.bb + 6 * (size_t)l;
    atomicMin(&b[0], z); atomicMax(&b[1], z); atomicMin(&b[2], y); atomicMax(&b[3], y); atomicMin(&b[4], x); atomicMax(&b[5], x);
}

// centroid sums: one warp per cluster over the box of its members, in raster order.
// Slab mode (xchg != null): the cluster is summed by the slab that owns the slice of the centre the assignment used; every member
// the assignment gave it lies within 2*step_z slices of that centre, i.e. inside the owner's k-means slab.  A member box that
// reaches beyond +- halo slices (a voxel no window reached kept the label of a cluster centred further away) is counted in
// xchg[5n]: the owner's sums would miss it.  The owner writes the record xchg[5k..5k+4] = bits(cz, cy, cx, cv), 1 (alive); every
// other slab, and the owner of a cluster that lost its last voxel, leaves zeros, so an integer sum over the slabs is an exact merge.
__global__ void __launch_bounds__(256) k3_update(Km3 s, const double* __restrict__ vol, const int* __restrict__ labels,
                                                 long long* __restrict__ xchg)
{
    __shared__ double buf[8][32];
    const int lane = threadIdx.x & 31, wl = threadIdx.x >> 5;
    const int k = blockIdx.x * 8 + wl;
    if (k >= s.n) return;
    const int* b = s.bb + 6 * (size_t)k;
    const int z0 = b[0], z1 = b[1], y0 = b[2], y1 = b[3], x0 = b[4], x1 = b[5];
    if (xchg) {
        const int cr = s.alive[k] ? (int)s.cz[k] : 0;   // slice of the centre the assignment used
        if (lane == 0 && z1 >= z0 && (!s.alive[k] || z0 < cr - s.halo || z1 > cr + s.halo))
            atomicAdd((unsigned long long*)&xchg[5 * (size_t)s.n], 1ull);
        if (!s.alive[k] || cr < s.own_lo || cr >= s.own_hi) return;
    } else if (!s.alive[k]) return;
    double acc = 0.0;
    long long cnt = 0, sumz = 0, sumy = 0, sumx = 0;
    for (int z = z0; z <= z1; ++z)
        for (int y = y0; y <= y1; ++y)
            for (int xb = x0; xb <= x1; xb += 32) {
                const int x = xb + lane;
                const size_t p = ((size_t)(z - s.z_off) * s.H + y) * s.W + x;
                const bool m = x <= x1 && labels[p] == k;
                const unsigned mask = __ballot_sync(0xffffffffu, m);
                if (!mask) continue;
                const int nm = __popc(mask);
                if (m) { buf[wl][__popc(mask & ((1u << lane) - 1u))] = vol[p]; sumx += x; }
                cnt += nm; sumz += (long long)z * nm; sumy += (long long)y * nm;
                __syncwarp();
                if (lane == 0) for (int i = 0; i < nm; ++i) acc = __dadd_rn(acc, buf[wl][i]);
                __syncwarp();
            }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sumx += __shfl_xor_sync(0xffffffffu, sumx, o);
    if (lane == 0) {
        if (cnt > 0) {
            const double dn = (double)cnt;
            const double cz = __ddiv_rn((double)sumz, dn), cy = __ddiv_rn((double)sumy, dn), cx = __ddiv_rn((double)sumx, dn);
            const double cv = __ddiv_rn(acc, dn);
            if (xchg) {
                long long* r = xchg + 5 * (size_t)k;
                r[0] = __double_as_longlong(cz); r[1] = __double_as_longlong(cy); r[2] = __double_as_longlong(cx);
                r[3] = __double_as_longlong(cv); r[4] = 1;
            } else { s.cz[k] = cz; s.cy[k] = cy; s.cx[k] = cx; s.cv[k] = cv; }
        } else if (!xchg) s.alive[k] = 0;   // no voxel: dead for good
    }
}

// slab mode: take the merged exchange records (see k3_update) as the replicated cluster state
__global__ void k3_import(Km3 s, const long long* __restrict__ xchg)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= s.n) return;
    const long long* r = xchg + 5 * (size_t)k;
    if (r[4] == 1) {
        s.cz[k] = __longlong_as_double(r[0]); s.cy[k] = __longlong_as_double(r[1]); s.cx[k] = __longlong_as_double(r[2]);
        s.cv[k] = __longlong_as_double(r[3]);
    } else s.alive[k] = 0;   // its owner found no voxel, or it was dead already (an alive cluster has exactly one owner)
}

__global__ void k3_fill(int* p, size_t n, int v)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

static size_t carve_km3(Km3& s, void* ws, size_t bytes, int D, int H, int W, int n)
{
    WsCarver c(ws, bytes);
    const size_t V = (size_t)D * H * W;
    s.cz = c.take<double>(n); s.cy = c.take<double>(n); s.cx = c.take<double>(n); s.cv = c.take<double>(n);
    s.alive = c.take<int>(n);
    s.bb = c.take<int>(6 * (size_t)n);
    s.dist = c.take<unsigned long long>(V);
    s.lab_new = c.take<int>(V);
    return isb_align(c.off);
}

// ---------------------------------------------------------------------------------------------------------------------
// connectivity
// ---------------------------------------------------------------------------------------------------------------------

struct Cc3 {
    int* parent;    // [V] union-find, then component root (first raster voxel)
    int* size;      // [V] component size at the root
    int* piece;     // [V] head voxel of the piece the voxel belongs to
    int* psize;     // [V] piece size at the head
    int* assigned;  // [V] split replay: voxel already in a piece / BFS replay of small pieces: voxel already queued
    int* adj;       // [V] at the head of a small piece: the piece it merges into (-1: label 0)
    int* newlab;    // [V] at the head of a kept piece: its label
    int* queue;     // [V] BFS queues: max_size entries per component >= max_size in the split (#big * max_size <= V), then
                    //     psize entries per small piece in their replay (sum of psize <= V); the split is done when the replay starts
    int* big;       // [V] roots of the components >= max_size
    int* counters;  // [0] #big, [1] queue cursor of the small-piece replay, [2] number of kept pieces
    int D, H, W;
};

__device__ __forceinline__ int find3(const int* parent, int x)
{
    while (true) { const int p = parent[x]; if (p == x) return x; x = p; }
}

__device__ __forceinline__ void unite3(int* parent, int a, int b)
{
    while (true) {
        a = find3(parent, a); b = find3(parent, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }   // hook the larger root under the smaller one
        const int old = atomicMin(&parent[a], b);
        if (old == a) return;
        a = old;
    }
}

__global__ void c3_init(Cc3 c)
{
    const size_t V = (size_t)c.D * c.H * c.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 3) c.counters[i] = 0;         // before the bound check: a volume of one or two voxels still clears all three
    if (i >= V) return;
    c.parent[i] = (int)i; c.size[i] = 0; c.psize[i] = 0; c.assigned[i] = 0; c.adj[i] = -1; c.newlab[i] = -1;
}

__global__ void c3_union(Cc3 c, const int* __restrict__ seg)
{
    const size_t V = (size_t)c.D * c.H * c.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    const int x = (int)(i % c.W), y = (int)((i / c.W) % c.H), z = (int)(i / ((size_t)c.H * c.W));
    const int l = seg[i];
    if (x + 1 < c.W && seg[i + 1] == l) unite3(c.parent, (int)i, (int)i + 1);
    if (y + 1 < c.H && seg[i + c.W] == l) unite3(c.parent, (int)i, (int)(i + c.W));
    if (z + 1 < c.D && seg[i + (size_t)c.H * c.W] == l) unite3(c.parent, (int)i, (int)(i + (size_t)c.H * c.W));
}

__global__ void c3_flatten(Cc3 c)
{
    const size_t V = (size_t)c.D * c.H * c.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    const int r = find3(c.parent, (int)i);
    c.piece[i] = r;                       // parent[] itself is flattened in the next kernel (other threads still walk it)
    atomicAdd(&c.size[r], 1);
}

__global__ void c3_collect(Cc3 c, int max_size)
{
    const size_t V = (size_t)c.D * c.H * c.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    c.parent[i] = c.piece[i];             // component root of every voxel
    if (c.piece[i] == (int)i && c.size[i] >= max_size) c.big[atomicAdd(&c.counters[0], 1)] = (int)i;
}

__device__ __forceinline__ int neighbour3(const Cc3& c, int v, int dir)
{
    // skimage's order: x+1, x-1, y+1, y-1, z+1, z-1
    const int x = v % c.W, y = (v / c.W) % c.H, z = v / (c.H * c.W);
    switch (dir) {
        case 0: return x + 1 < c.W ? v + 1 : -1;
        case 1: return x > 0 ? v - 1 : -1;
        case 2: return y + 1 < c.H ? v + c.W : -1;
        case 3: return y > 0 ? v - c.W : -1;
        case 4: return z + 1 < c.D ? v + c.H * c.W : -1;
        default: return z > 0 ? v - c.H * c.W : -1;
    }
}

// one thread per component >= max_size: replay the raster scan + truncated BFS of the original on that component alone
__global__ void c3_split(Cc3 c, int max_size)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= c.counters[0]) return;
    const int root = c.big[t];
    const int V = c.D * c.H * c.W;
    int* q = c.queue + (size_t)t * max_size;   // the component's own queue, reused by each of its pieces
    int remaining = c.size[root];
    int scan = root;
    while (remaining > 0) {
        while (scan < V && !(c.parent[scan] == root && c.assigned[scan] == 0)) ++scan;
        if (scan >= V) break;
        const int head = scan;
        c.assigned[head] = 1; c.piece[head] = head; q[0] = head;
        int size = 1, visited = 0;
        while (visited < size && size < max_size) {
            const int u = q[visited];
            for (int dir = 0; dir < 6; ++dir) {
                const int n = neighbour3(c, u, dir);
                if (n >= 0 && c.parent[n] == root && c.assigned[n] == 0) {
                    c.assigned[n] = 1; c.piece[n] = head; q[size] = n;
                    size += 1;
                    if (size >= max_size) break;
                }
            }
            visited += 1;
        }
        remaining -= size;
        scan = head + 1;
    }
}

__global__ void c3_piece_sizes(Cc3 c)
{
    const size_t V = (size_t)c.D * c.H * c.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= V) return;
    atomicAdd(&c.psize[c.piece[i]], 1);
    c.assigned[i] = 0;    // reused as the "queued" flag of the small-piece replay
}

// labels of the kept pieces: rank of their head voxel among the kept heads, in raster order (single CTA, chunked scan)
__global__ void __launch_bounds__(1024) c3_rank(Cc3 c, int min_size)
{
    const auto kept_head = [&](int i) { return c.piece[i] == i && c.psize[i] >= min_size; };
    const int total = cta_scan_chunks<1024, int>(c.D * c.H * c.W, [&](int i) { return kept_head(i) ? 1 : 0; },
                                                 [&](int i, int rank) { if (kept_head(i)) c.newlab[i] = rank; });
    if (threadIdx.x == 0) c.counters[2] = total;
}

// one thread per small piece: replay its BFS to find the LAST neighbour that belongs to an earlier piece
__global__ void c3_small(Cc3 c, int min_size)
{
    const int V = c.D * c.H * c.W;
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= V || c.piece[h] != h || c.psize[h] >= min_size) return;
    int* q = c.queue + atomicAdd(&c.counters[1], c.psize[h]);
    int adj = -1;
    c.assigned[h] = 1; q[0] = h;
    int size = 1, visited = 0;
    while (visited < size) {
        const int u = q[visited];
        for (int dir = 0; dir < 6; ++dir) {
            const int n = neighbour3(c, u, dir);
            if (n < 0) continue;
            const int pn = c.piece[n];
            if (pn == h) { if (!c.assigned[n]) { c.assigned[n] = 1; q[size++] = n; } }
            else if (pn < h) adj = pn;      // labelled before this piece started
        }
        visited += 1;
    }
    c.adj[h] = adj;
}

__global__ void c3_write(Cc3 c, int min_size, int* __restrict__ out, int* __restrict__ n_labels)
{
    const size_t V = (size_t)c.D * c.H * c.W;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *n_labels = c.counters[2] > 0 ? c.counters[2] : 1;
    if (i >= V) return;
    int h = c.piece[i];
    while (h >= 0 && c.psize[h] < min_size) h = c.adj[h];     // small pieces chain to earlier pieces
    out[i] = h >= 0 ? c.newlab[h] : 0;                         // no earlier neighbour at all: the original's default label 0
}

static size_t carve_cc3(Cc3& c, void* ws, size_t bytes, int D, int H, int W)
{
    WsCarver w(ws, bytes);
    const size_t V = (size_t)D * H * W;
    c.D = D; c.H = H; c.W = W;
    c.parent = w.take<int>(V); c.size = w.take<int>(V); c.piece = w.take<int>(V); c.psize = w.take<int>(V);
    c.assigned = w.take<int>(V); c.adj = w.take<int>(V); c.newlab = w.take<int>(V);
    c.queue = w.take<int>(V);
    c.big = w.take<int>(V);
    c.counters = w.take<int>(4);
    return isb_align(w.off);
}

} // namespace

extern "C" int isb_slic3d_prepare_slab(const void* vol, int dtype, int S, int H, int W, int z_off, int D, const double* w_z, int r_z,
                                       const double* w_y, int r_y, const double* w_x, int r_x, double ratio, double* tmp, double* out,
                                       isb_stream_t stream)
{
    ISB_REQUIRE(vol && w_z && w_y && w_x && tmp && out, "null pointer");
    ISB_REQUIRE(S > 0 && H > 0 && W > 0 && r_z >= 0 && r_y >= 0 && r_x >= 0, "bad sizes");
    ISB_REQUIRE(z_off >= 0 && z_off + S <= D, "slab outside the volume");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)S * H * W;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    k3_load<<<blocks, 256, 0, st>>>(vol, dtype, n, out);
    ISB_LAUNCH_CHECK();
    k3_blur_axis<<<blocks, 256, 0, st>>>(out, tmp, S, H, W, z_off, D, 0, w_z, r_z);
    ISB_LAUNCH_CHECK();
    k3_blur_axis<<<blocks, 256, 0, st>>>(tmp, out, S, H, W, z_off, D, 1, w_y, r_y);
    ISB_LAUNCH_CHECK();
    k3_blur_axis<<<blocks, 256, 0, st>>>(out, tmp, S, H, W, z_off, D, 2, w_x, r_x);
    ISB_LAUNCH_CHECK();
    // image * ratio is its own rounding step (np.ascontiguousarray(image * ratio))
    k3_scale<<<blocks, 256, 0, st>>>(tmp, out, n, ratio);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_slic3d_prepare(const void* vol, int dtype, int D, int H, int W, const double* w_z, int r_z, const double* w_y, int r_y,
                                  const double* w_x, int r_x, double ratio, double* tmp, double* out, isb_stream_t stream)
{
    return isb_slic3d_prepare_slab(vol, dtype, D, H, W, 0, D, w_z, r_z, w_y, r_y, w_x, r_x, ratio, tmp, out, stream);
}

extern "C" size_t isb_slic3d_kmeans_workspace_bytes(int D, int H, int W, int n_seeds)
{
    Km3 s;
    return carve_km3(s, nullptr, 0, D, H, W, n_seeds);
}

extern "C" int isb_slic3d_kmeans(const double* vol_scaled, int D, int H, int W, const double* seeds_zyx, int n_seeds, int step_z, int step_y,
                                 int step_x, double step, const double* spacing_host, int max_iter, int32_t* labels, void* ws,
                                 size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(vol_scaled && seeds_zyx && spacing_host && labels && ws, "null pointer");
    ISB_REQUIRE(D > 0 && H > 0 && W > 0 && n_seeds > 0 && step_z > 0 && step_y > 0 && step_x > 0 && step > 0, "bad sizes");
    ISB_REQUIRE((size_t)D * H * W < (size_t)INT_MAX, "volume too large");
    Km3 s;
    const size_t need = carve_km3(s, ws, ws_bytes, D, H, W, n_seeds);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    s.n = n_seeds; s.D = D; s.H = H; s.W = W; s.step_z = step_z; s.step_y = step_y; s.step_x = step_x;
    s.z_off = 0; s.Dg = D; s.own_lo = 0; s.own_hi = D; s.halo = D;
    s.sz = spacing_host[0]; s.sy = spacing_host[1]; s.sx = spacing_host[2]; s.sw = 1.0 / (step * step);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t V = (size_t)D * H * W;
    const size_t m = V > (size_t)n_seeds ? V : (size_t)n_seeds;
    const unsigned vblocks = (unsigned)((V + 255) / 256), mblocks = (unsigned)((m + 255) / 256);
    k3_fill<<<vblocks, 256, 0, st>>>(labels, V, 0);
    ISB_LAUNCH_CHECK();
    k3_seed<<<(n_seeds + 255) / 256, 256, 0, st>>>(s, seeds_zyx);
    ISB_LAUNCH_CHECK();
    for (int it = 0; it < max_iter; ++it) {
        k3_clear<<<mblocks, 256, 0, st>>>(s);
        ISB_LAUNCH_CHECK();
        k3_scan<0><<<n_seeds, 256, 0, st>>>(s, vol_scaled);
        ISB_LAUNCH_CHECK();
        k3_scan<1><<<n_seeds, 256, 0, st>>>(s, vol_scaled);
        ISB_LAUNCH_CHECK();
        k3_commit<<<vblocks, 256, 0, st>>>(s, labels);
        ISB_LAUNCH_CHECK();
        k3_update<<<(n_seeds + 7) / 8, 256, 0, st>>>(s, vol_scaled, labels, nullptr);
        ISB_LAUNCH_CHECK();
    }
    return ISB_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Slab mode: the same sweeps with one z-slab of the volume per GPU.  The cluster state is replicated; what crosses the GPUs
// each sweep is the exchange buffer of k3_update (summed as int64 by the caller's collective).
// ---------------------------------------------------------------------------------------------------------------------
namespace {

static int slab_state(const isb_slic3d_slab_t* b, Km3& s)
{
    ISB_REQUIRE(b && b->vol_slab && b->seeds_zyx && b->labels_slab && b->ws, "null pointer");
    ISB_REQUIRE(b->depth > 0 && b->height > 0 && b->width > 0 && b->slab_slices > 0 && b->n_seeds > 0 && b->step_z > 0 && b->step_y > 0 &&
                b->step_x > 0 && b->step > 0, "bad sizes");
    ISB_REQUIRE((size_t)b->depth * b->height * b->width < (size_t)INT_MAX, "volume too large");
    ISB_REQUIRE(b->z_off >= 0 && b->z_off + b->slab_slices <= b->depth, "slab outside the volume");
    ISB_REQUIRE(b->own_lo >= b->z_off && b->own_hi <= b->z_off + b->slab_slices && b->own_lo < b->own_hi, "owned slices outside the slab");
    ISB_REQUIRE(b->halo >= 2 * b->step_z, "halo must be at least 2 * step_z slices");
    ISB_REQUIRE(b->z_off <= (b->own_lo - b->halo > 0 ? b->own_lo - b->halo : 0), "slab does not cover the halo below the owned slices");
    ISB_REQUIRE(b->z_off + b->slab_slices >= (b->own_hi + b->halo < b->depth ? b->own_hi + b->halo : b->depth),
                "slab does not cover the halo above the owned slices");
    const size_t need = carve_km3(s, b->ws, b->ws_bytes, b->slab_slices, b->height, b->width, b->n_seeds);
    ISB_REQUIRE(need <= b->ws_bytes, "workspace too small");
    s.n = b->n_seeds; s.D = b->slab_slices; s.H = b->height; s.W = b->width;
    s.step_z = b->step_z; s.step_y = b->step_y; s.step_x = b->step_x;
    s.z_off = b->z_off; s.Dg = b->depth; s.own_lo = b->own_lo; s.own_hi = b->own_hi; s.halo = b->halo;
    s.sz = b->spacing[0]; s.sy = b->spacing[1]; s.sx = b->spacing[2]; s.sw = 1.0 / (b->step * b->step);
    return ISB_OK;
}

} // namespace

extern "C" int isb_slic3d_slab_begin(const isb_slic3d_slab_t* b, isb_stream_t stream)
{
    Km3 s;
    if (int rc = slab_state(b, s)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t V = (size_t)s.D * s.H * s.W;
    k3_fill<<<(unsigned)((V + 255) / 256), 256, 0, st>>>(b->labels_slab, V, 0);
    ISB_LAUNCH_CHECK();
    k3_seed<<<(s.n + 255) / 256, 256, 0, st>>>(s, b->seeds_zyx);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_slic3d_slab_assign(const isb_slic3d_slab_t* b, isb_stream_t stream)
{
    Km3 s;
    if (int rc = slab_state(b, s)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t V = (size_t)s.D * s.H * s.W;
    const size_t m = V > (size_t)s.n ? V : (size_t)s.n;
    k3_clear<<<(unsigned)((m + 255) / 256), 256, 0, st>>>(s);
    ISB_LAUNCH_CHECK();
    k3_scan<0><<<s.n, 256, 0, st>>>(s, b->vol_slab);
    ISB_LAUNCH_CHECK();
    k3_scan<1><<<s.n, 256, 0, st>>>(s, b->vol_slab);
    ISB_LAUNCH_CHECK();
    k3_commit<<<(unsigned)((V + 255) / 256), 256, 0, st>>>(s, b->labels_slab);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_slic3d_slab_update(const isb_slic3d_slab_t* b, int64_t* xchg, isb_stream_t stream)
{
    Km3 s;
    if (int rc = slab_state(b, s)) return rc;
    ISB_REQUIRE(xchg, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    ISB_CUDA_CHECK(cudaMemsetAsync(xchg, 0, sizeof(int64_t) * (5 * (size_t)s.n + 1), st));
    k3_update<<<(s.n + 7) / 8, 256, 0, st>>>(s, b->vol_slab, b->labels_slab, (long long*)xchg);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_slic3d_slab_import(const isb_slic3d_slab_t* b, const int64_t* xchg, isb_stream_t stream)
{
    Km3 s;
    if (int rc = slab_state(b, s)) return rc;
    ISB_REQUIRE(xchg, "null pointer");
    k3_import<<<(s.n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(s, (const long long*)xchg);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" size_t isb_connectivity3d_workspace_bytes(int D, int H, int W, int max_size)
{
    Cc3 c;
    (void)max_size;                       // the queues fit in V entries whatever max_size is
    return carve_cc3(c, nullptr, 0, D, H, W);
}

extern "C" int isb_enforce_connectivity3d(const int32_t* labels, int D, int H, int W, int min_size, int max_size, int32_t* out,
                                          int32_t* n_labels_out, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(labels && out && n_labels_out && ws, "null pointer");
    ISB_REQUIRE(D > 0 && H > 0 && W > 0, "bad sizes");
    ISB_REQUIRE((size_t)D * H * W < (size_t)INT_MAX / 4, "volume too large");
    if (max_size < 1) max_size = 1;
    Cc3 c;
    const size_t need = carve_cc3(c, ws, ws_bytes, D, H, W);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t V = (size_t)D * H * W;
    const unsigned vblocks = (unsigned)((V + 255) / 256);
    c3_init<<<vblocks, 256, 0, st>>>(c);
    ISB_LAUNCH_CHECK();
    c3_union<<<vblocks, 256, 0, st>>>(c, labels);
    ISB_LAUNCH_CHECK();
    c3_flatten<<<vblocks, 256, 0, st>>>(c);
    ISB_LAUNCH_CHECK();
    c3_collect<<<vblocks, 256, 0, st>>>(c, max_size);
    ISB_LAUNCH_CHECK();
    c3_split<<<vblocks, 256, 0, st>>>(c, max_size);       // as many threads as there could be oversize components
    ISB_LAUNCH_CHECK();
    c3_piece_sizes<<<vblocks, 256, 0, st>>>(c);
    ISB_LAUNCH_CHECK();
    c3_rank<<<1, 1024, 0, st>>>(c, min_size);
    ISB_LAUNCH_CHECK();
    c3_small<<<vblocks, 256, 0, st>>>(c, min_size);
    ISB_LAUNCH_CHECK();
    c3_write<<<vblocks, 256, 0, st>>>(c, min_size, out, n_labels_out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
