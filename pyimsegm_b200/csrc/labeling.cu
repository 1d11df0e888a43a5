// labeling.cu -- the label-map kernels of the reference's imsegm/labeling.py:
//   thick boundary map   (skimage find_boundaries(mode='thick') inside compute_boundary_distances :684-716)
//   interior contour map (contour_binary_map :34-79, contour_coords :82-117)
//   exact 2-D Euclidean distance transform (scipy.ndimage.distance_transform_edt, compute_distance_map :146-169), and the same transform
//   giving the index of a nearest site (distance_transform_edt(..., return_indices=True); image_inpaint_pixels of annotation.py)
//   order-preserving mask compaction (the (row, col) lists of contour_coords and compute_boundary_distances)
//   relabel gather with negative pass-through (relabel_max_overlap_unique :611-613, relabel_max_overlap_merge :678-680)
// The overlap matrix (compute_labels_overlap_matrix :490-523) is isb_region_label_hist (native_misc.cu).
#include "compact.cuh"

namespace {

// ---------------------------------------------------------------------------------------------------------------------
// boundary and contour maps
// ---------------------------------------------------------------------------------------------------------------------

// grey_dilation(l, cross) != grey_erosion(l, cross) with scipy's 'reflect' border: p is on the boundary iff one of its in-image
// 4-neighbours carries a different label
__global__ void __launch_bounds__(256) k_thick_boundary(const int* __restrict__ seg, int H, int W, uint8_t* __restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)H * W) return;
    const int y = (int)(i / W), x = (int)(i % W);
    const int l = seg[i];
    bool b = (x > 0 && seg[i - 1] != l) || (x + 1 < W && seg[i + 1] != l);
    b = b || (y > 0 && seg[i - W] != l) || (y + 1 < H && seg[i + W] != l);
    out[i] = b ? 1 : 0;
}

// contour_binary_map: rows 1..H-2 and columns 1..W-2 are set where the label has a 4-neighbour of another label; with
// include_boundary every pixel of the label on the outer frame as well
__global__ void __launch_bounds__(256) k_contour(const int* __restrict__ seg, int H, int W, int label, int include_boundary,
                                                 uint8_t* __restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)H * W) return;
    const int y = (int)(i / W), x = (int)(i % W);
    const bool on = seg[i] == label;
    const bool frame = y == 0 || y == H - 1 || x == 0 || x == W - 1;
    bool v;
    if (frame) v = on && include_boundary;
    else v = on && (seg[i - 1] != label || seg[i + 1] != label || seg[i - W] != label || seg[i + W] != label);
    out[i] = v ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// exact EDT, banded in both phases as in the Parallel Banding Algorithm (Cao et al., 2010).
// Phase 1 runs down the columns in bands of 32 rows and writes the column distance g transposed, gT[x][y], so that every phase-2
// kernel below walks one image row per thread with consecutive threads on consecutive rows (coalesced).
// Phase 2 takes per row the lower envelope of the parabolas (x - u)^2 + g(u)^2 over the real line: each band of 32 columns builds the
// envelope of its own sites as a doubly linked list (prev / next, stored at the site's column), neighbouring bands are merged pairwise
// in log2(bands) launches (the union's envelope is a prefix of the left list followed by a suffix of the right one, so a merge only
// touches the junction), every surviving site marks the first column it owns, and a banded prefix maximum of the marks gives each
// pixel its nearest site.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int EDT_BAND = 32;     // rows per phase-1 band: one bit each in a 32-bit word
constexpr int EDT_COLS = 32;     // columns per phase-2 band
constexpr int EDT_ROWS = 128;    // rows (threads) per phase-2 CTA
constexpr int EDT_NONE = 0x7fffffff;
constexpr int EDT_DEAD = -2;     // prev[] of a column that is not on the envelope (no site, or dominated)

// 1a: the sites of every (band, column) as a bit word (bit r = row band*32 + r)
__global__ void __launch_bounds__(256) k_edt_bits(const uint8_t* __restrict__ sites, int H, int W, unsigned* __restrict__ bits)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (x >= W) return;
    const int y0 = b * EDT_BAND, y1 = min(y0 + EDT_BAND, H);
    unsigned m = 0;
    for (int y = y0; y < y1; ++y) m |= (sites[(size_t)y * W + x] != 0 ? 1u : 0u) << (y - y0);
    bits[(size_t)b * W + x] = m;
}

// 1b: per column, the last site row above each band and the first site row below it (-1 / EDT_NONE when there is none)
__global__ void __launch_bounds__(256) k_edt_links(const unsigned* __restrict__ bits, int nb, int W, int* __restrict__ above,
                                                   int* __restrict__ below)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= W) return;
    int last = -1;
    for (int b = 0; b < nb; ++b) {
        above[(size_t)b * W + x] = last;
        const unsigned m = bits[(size_t)b * W + x];
        if (m) last = b * EDT_BAND + 31 - __clz(m);
    }
    int first = EDT_NONE;
    for (int b = nb - 1; b >= 0; --b) {
        below[(size_t)b * W + x] = first;
        const unsigned m = bits[(size_t)b * W + x];
        if (m) first = b * EDT_BAND + __ffs(m) - 1;
    }
}

// 1c: gT[x][y] = distance from (y, x) to the nearest site in column x (EDT_NONE for a column without one), transposed through
// shared memory so that both the reads and the writes are coalesced.  IDX (the nearest-site variant) also writes upT[x][y] = 1 when
// that site lies above (row y - gT), 0 when below (row y + gT); equidistant sites above and below give the upper one.
template <bool IDX>
__global__ void __launch_bounds__(256) k_edt_cols(const unsigned* __restrict__ bits, const int* __restrict__ above,
                                                  const int* __restrict__ below, int H, int W, int* __restrict__ gT,
                                                  uint8_t* __restrict__ upT)
{
    __shared__ int tile[EDT_BAND][256 + 1];
    __shared__ uint8_t up_tile[IDX ? EDT_BAND : 1][IDX ? 256 + 4 : 1];
    const int xb = blockIdx.x * 256, x = xb + threadIdx.x, b = blockIdx.y;
    const int y0 = b * EDT_BAND, y1 = min(y0 + EDT_BAND, H);
    if (x < W) {
        const size_t k = (size_t)b * W + x;
        const unsigned m = bits[k];
        const int up = above[k], dn = below[k];
        for (int y = y0; y < y1; ++y) {
            const int r = y - y0;
            const unsigned upto = m & (0xffffffffu >> (31 - r));        // sites at rows y0 .. y
            const unsigned from = m & (0xffffffffu << r);               // sites at rows y .. y0 + 31
            const int a = upto ? y0 + 31 - __clz(upto) : up;
            const int c = from ? y0 + __ffs(from) - 1 : dn;
            int d = EDT_NONE;
            if (a >= 0) d = y - a;
            if (c != EDT_NONE) d = min(d, c - y);
            tile[r][threadIdx.x] = d;
            if constexpr (IDX) up_tile[r][threadIdx.x] = a >= 0 && y - a == d;
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < 256 * EDT_BAND; e += 256) {
        const int xx = e / EDT_BAND, r = e % EDT_BAND;
        if (xb + xx < W && y0 + r < y1) {
            gT[(size_t)(xb + xx) * H + y0 + r] = tile[r][xx];
            if constexpr (IDX) upT[(size_t)(xb + xx) * H + y0 + r] = up_tile[r][xx];
        }
    }
}

__device__ __forceinline__ long long parab(int x, int u, int gu) { return (long long)(x - u) * (x - u) + (long long)gu * gu; }

// numerator of the abscissa where the parabolas of sites a < b cross: x_ab = num / (2 (b - a))
__device__ __forceinline__ long long cross_num(int a, int ga, int b, int gb)
{
    return (long long)b * b - (long long)a * a + (long long)gb * gb - (long long)ga * ga;
}

// b (a < b < c) owns no part of the real line: x_ab >= x_bc, compared exactly (|num| < 2^32, spans < 2^15)
__device__ __forceinline__ bool dominated(int a, int ga, int b, int gb, int c, int gc)
{
    return cross_num(a, ga, b, gb) * (c - b) >= cross_num(b, gb, c, gc) * (b - a);
}

// first integer column strictly right of x_ab, clamped to [-1, W]
__device__ __forceinline__ int first_after(int a, int ga, int b, int gb, int W)
{
    const long long num = cross_num(a, ga, b, gb), den = 2LL * (b - a);
    long long q = num / den;
    if (num % den != 0 && num < 0) --q;                 // floor division
    return (int)max(-1LL, min((long long)W, q + 1));
}

// 2a: per (row, band of EDT_COLS columns) the envelope of the band's own sites; head / tail of the list per (band, row)
__global__ void __launch_bounds__(EDT_ROWS) k_edt_local(const int* __restrict__ gT, int H, int W, int* __restrict__ prev, int* __restrict__ next,
                                                        int* __restrict__ head, int* __restrict__ tail)
{
    const int y = blockIdx.x * EDT_ROWS + threadIdx.x, b = blockIdx.y;
    if (y >= H) return;
    const int x0 = b * EDT_COLS, x1 = min(x0 + EDT_COLS, W);
    int top = -1, gt = 0, below = -1, gb = 0;
    for (int u = x0; u < x1; ++u) {
        const int gu = gT[(size_t)u * H + y];
        if (gu == EDT_NONE) { prev[(size_t)u * H + y] = EDT_DEAD; continue; }
        while (below >= 0 && dominated(below, gb, top, gt, u, gu)) {
            prev[(size_t)top * H + y] = EDT_DEAD;
            top = below; gt = gb;
            below = prev[(size_t)top * H + y];
            if (below >= 0) gb = gT[(size_t)below * H + y];
        }
        prev[(size_t)u * H + y] = top;
        below = top; gb = gt; top = u; gt = gu;
    }
    int h = -1;
    for (int v = top, n = -1; v >= 0; n = v, v = prev[(size_t)v * H + y]) { next[(size_t)v * H + y] = n; h = v; }
    head[(size_t)b * H + y] = h;
    tail[(size_t)b * H + y] = top;
}

// 2b: merge the lists of band groups [2jG, 2jG + G) and [2jG + G, 2jG + 2G) of one row; the result is kept at the left group's index
__global__ void __launch_bounds__(EDT_ROWS) k_edt_merge(const int* __restrict__ gT, int H, int nb, int G, int* __restrict__ prev,
                                                        int* __restrict__ next, int* __restrict__ head, int* __restrict__ tail)
{
    const int y = blockIdx.x * EDT_ROWS + threadIdx.x, bl = 2 * blockIdx.y * G, br = bl + G;
    if (y >= H || br >= nb) return;
    const size_t L = (size_t)bl * H + y, R = (size_t)br * H + y;
    const int rh = head[R];
    if (rh < 0) return;
    const int lt = tail[L];
    if (lt < 0) { head[L] = rh; tail[L] = tail[R]; return; }
    int l1 = lt, g1 = gT[(size_t)l1 * H + y], l0 = prev[(size_t)l1 * H + y], g0 = l0 >= 0 ? gT[(size_t)l0 * H + y] : 0;
    int r0 = rh, h0 = gT[(size_t)r0 * H + y], r1 = next[(size_t)r0 * H + y], h1 = r1 >= 0 ? gT[(size_t)r1 * H + y] : 0;
    for (;;) {
        if (l0 >= 0 && dominated(l0, g0, l1, g1, r0, h0)) {
            prev[(size_t)l1 * H + y] = EDT_DEAD;
            l1 = l0; g1 = g0;
            l0 = prev[(size_t)l1 * H + y];
            if (l0 >= 0) g0 = gT[(size_t)l0 * H + y];
            continue;
        }
        if (r1 >= 0 && dominated(l1, g1, r0, h0, r1, h1)) {
            prev[(size_t)r0 * H + y] = EDT_DEAD;
            r0 = r1; h0 = h1;
            r1 = next[(size_t)r0 * H + y];
            if (r1 >= 0) h1 = gT[(size_t)r1 * H + y];
            continue;
        }
        break;
    }
    next[(size_t)l1 * H + y] = r0;
    prev[(size_t)r0 * H + y] = l1;
    tail[L] = tail[R];
}

// 2c: every site on the row's envelope writes its column at the first column it owns (owned ranges are disjoint: plain stores)
__global__ void __launch_bounds__(EDT_ROWS) k_edt_marks(const int* __restrict__ gT, const int* __restrict__ prev, const int* __restrict__ next,
                                                        int H, int W, int* __restrict__ mark)
{
    const int y = blockIdx.x * EDT_ROWS + threadIdx.x, b = blockIdx.y;
    if (y >= H) return;
    const int x0 = b * EDT_COLS, x1 = min(x0 + EDT_COLS, W);
    for (int u = x0; u < x1; ++u) {
        const int p = prev[(size_t)u * H + y];
        if (p == EDT_DEAD) continue;
        const int gu = gT[(size_t)u * H + y], n = next[(size_t)u * H + y];
        const int lo = max(0, p < 0 ? 0 : first_after(p, gT[(size_t)p * H + y], u, gu, W));
        const int hi = n < 0 ? W : first_after(u, gu, n, gT[(size_t)n * H + y], W);
        if (lo < hi) mark[(size_t)lo * H + y] = u;
    }
}

// 2d: largest mark of every (band, row), then per row the largest mark left of each band
__global__ void __launch_bounds__(EDT_ROWS) k_edt_bandmax(const int* __restrict__ mark, int H, int W, int* __restrict__ bmax)
{
    const int y = blockIdx.x * EDT_ROWS + threadIdx.x, b = blockIdx.y;
    if (y >= H) return;
    const int x0 = b * EDT_COLS, x1 = min(x0 + EDT_COLS, W);
    int m = -1;
    for (int x = x0; x < x1; ++x) m = max(m, mark[(size_t)x * H + y]);
    bmax[(size_t)b * H + y] = m;
}

__global__ void __launch_bounds__(EDT_ROWS) k_edt_carry(const int* __restrict__ bmax, int H, int nb, int* __restrict__ carry)
{
    const int y = blockIdx.x * EDT_ROWS + threadIdx.x;
    if (y >= H) return;
    int c = -1;
    for (int b = 0; b < nb; ++b) {
        carry[(size_t)b * H + y] = c;
        c = max(c, bmax[(size_t)b * H + y]);
    }
}

// 2e: the nearest site of every pixel is the running maximum of the marks; dist = sqrt((double)d2) as scipy forms it, written row-major
// through shared memory.  A row without marks has no site anywhere in the image: scipy then measures every pixel from (-1, 0).
// IDX writes instead the flat index (row * W + column) of that site, its row from upT, or -1 when the image has no site.
template <bool IDX> struct EdtOut { using T = double; };
template <> struct EdtOut<true> { using T = int; };

template <bool IDX>
__global__ void __launch_bounds__(EDT_ROWS) k_edt_fill(const int* __restrict__ gT, const int* __restrict__ mark, const int* __restrict__ carry,
                                                       const uint8_t* __restrict__ upT, int H, int W, typename EdtOut<IDX>::T* __restrict__ out)
{
    __shared__ typename EdtOut<IDX>::T tile[EDT_ROWS][EDT_COLS + 1];
    const int b = blockIdx.x, y0 = blockIdx.y * EDT_ROWS, x0 = b * EDT_COLS, y = y0 + threadIdx.x;
    if (y < H) {
        int owner = carry[(size_t)b * H + y];
        int gown = owner >= 0 ? gT[(size_t)owner * H + y] : 0;
        for (int c = 0; c < EDT_COLS && x0 + c < W; ++c) {
            const int x = x0 + c, m = mark[(size_t)x * H + y];
            if (m > owner) { owner = m; gown = gT[(size_t)m * H + y]; }
            if constexpr (IDX) {
                tile[threadIdx.x][c] = owner >= 0 ? (upT[(size_t)owner * H + y] ? y - gown : y + gown) * W + owner : -1;
            } else {
                tile[threadIdx.x][c] = owner >= 0 ? sqrt((double)parab(x, owner, gown))
                                                  : sqrt((double)((long long)(y + 1) * (y + 1) + (long long)x * x));
            }
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < EDT_ROWS * EDT_COLS; e += EDT_ROWS) {
        const int r = e / EDT_COLS, c = e % EDT_COLS;
        if (y0 + r < H && x0 + c < W) out[(size_t)(y0 + r) * W + x0 + c] = tile[r][c];
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// order-preserving compaction of a [H, W] mask (compact.cuh): the writes in raster order
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CPT_THREADS) k_compact_write(const uint8_t* __restrict__ mask, long long n, int W, const double* __restrict__ values,
                                                               const long long* __restrict__ tile_off, int64_t* __restrict__ points,
                                                               double* __restrict__ values_out)
{
    const long long beg = (long long)blockIdx.x * CPT_TILE + (long long)threadIdx.x * CPT_PER;
    int total;
    long long o = tile_off[blockIdx.x] + cta_exclusive_sum<CPT_THREADS>(thread_count(mask, beg, n), total);
    for (int k = 0; k < CPT_PER; ++k) {
        const long long i = beg + k;
        if (i < n && mask[i]) {
            points[2 * o] = i / W;
            points[2 * o + 1] = i % W;
            if (values) values_out[o] = values[i];
            ++o;
        }
    }
}

__global__ void __launch_bounds__(256) k_relabel(const int* __restrict__ seg, long long n, const int* __restrict__ lut, int n_lut, int* __restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = seg[i];
    out[i] = (s >= 0 && s < n_lut) ? lut[s] : s;
}

inline int edt_bands(int H) { return (H + EDT_BAND - 1) / EDT_BAND; }
inline int edt_col_bands(int W) { return (W + EDT_COLS - 1) / EDT_COLS; }

} // namespace

extern "C" int isb_label_boundary_map(const int32_t* seg, int H, int W, uint8_t* out, isb_stream_t stream)
{
    ISB_REQUIRE(seg && out, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0, "bad sizes");
    const long long n = (long long)H * W;
    k_thick_boundary<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(seg, H, W, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_label_contour_map(const int32_t* seg, int H, int W, int32_t label, int include_boundary, uint8_t* out, isb_stream_t stream)
{
    ISB_REQUIRE(seg && out, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0, "bad sizes");
    const long long n = (long long)H * W;
    k_contour<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(seg, H, W, label, include_boundary ? 1 : 0, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" size_t isb_edt_workspace_bytes(int H, int W)
{
    if (H <= 0 || W <= 0) return 0;
    const size_t px = (size_t)H * W, bw = (size_t)edt_bands(H) * W, bh = (size_t)edt_col_bands(W) * H;
    return isb_align(sizeof(unsigned) * bw) + 2 * isb_align(sizeof(int) * bw) + 4 * isb_align(sizeof(int) * px) + 5 * isb_align(sizeof(int) * bh);
}

// both transforms share every kernel; IDX adds the above / below flags of the column pass and writes site indices instead of distances
template <bool IDX>
int edt_run(const uint8_t* sites, int H, int W, typename EdtOut<IDX>::T* out, void* ws, size_t ws_bytes, cudaStream_t st)
{
    const int nb = edt_bands(H), nc = edt_col_bands(W);
    WsCarver c(ws, ws_bytes);
    unsigned* bits = c.take<unsigned>((size_t)nb * W);
    int* above = c.take<int>((size_t)nb * W);
    int* below = c.take<int>((size_t)nb * W);
    int* gT = c.take<int>((size_t)H * W);
    int* prev = c.take<int>((size_t)H * W);
    int* next = c.take<int>((size_t)H * W);
    int* mark = c.take<int>((size_t)H * W);
    int* head = c.take<int>((size_t)nc * H);
    int* tail = c.take<int>((size_t)nc * H);
    int* bmax = c.take<int>((size_t)nc * H);
    int* carry = c.take<int>((size_t)nc * H);
    uint8_t* upT = IDX ? c.take<uint8_t>((size_t)H * W) : nullptr;
    const unsigned gx = (unsigned)((W + 255) / 256), gy = (unsigned)((H + EDT_ROWS - 1) / EDT_ROWS);
    k_edt_bits<<<dim3(gx, nb), 256, 0, st>>>(sites, H, W, bits);
    ISB_LAUNCH_CHECK();
    k_edt_links<<<gx, 256, 0, st>>>(bits, nb, W, above, below);
    ISB_LAUNCH_CHECK();
    k_edt_cols<IDX><<<dim3(gx, nb), 256, 0, st>>>(bits, above, below, H, W, gT, upT);
    ISB_LAUNCH_CHECK();
    k_edt_local<<<dim3(gy, nc), EDT_ROWS, 0, st>>>(gT, H, W, prev, next, head, tail);
    ISB_LAUNCH_CHECK();
    for (int G = 1; G < nc; G *= 2) {
        k_edt_merge<<<dim3(gy, (nc + 2 * G - 1) / (2 * G)), EDT_ROWS, 0, st>>>(gT, H, nc, G, prev, next, head, tail);
        ISB_LAUNCH_CHECK();
    }
    ISB_CUDA_CHECK(cudaMemsetAsync(mark, 0xff, sizeof(int) * (size_t)H * W, st));      // -1: no site starts here
    k_edt_marks<<<dim3(gy, nc), EDT_ROWS, 0, st>>>(gT, prev, next, H, W, mark);
    ISB_LAUNCH_CHECK();
    k_edt_bandmax<<<dim3(gy, nc), EDT_ROWS, 0, st>>>(mark, H, W, bmax);
    ISB_LAUNCH_CHECK();
    k_edt_carry<<<gy, EDT_ROWS, 0, st>>>(bmax, H, nc, carry);
    ISB_LAUNCH_CHECK();
    k_edt_fill<IDX><<<dim3(nc, gy), EDT_ROWS, 0, st>>>(gT, mark, carry, upT, H, W, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_edt_2d(const uint8_t* sites, int H, int W, double* dist, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(sites && dist && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0, "bad sizes");
    ISB_REQUIRE(H <= 32768 && W <= 32768, "the squared distances of an image larger than 32768 x 32768 overflow int32");
    ISB_REQUIRE(ws_bytes >= isb_edt_workspace_bytes(H, W), "workspace too small");
    return edt_run<false>(sites, H, W, dist, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t isb_edt_index_workspace_bytes(int H, int W)
{
    if (H <= 0 || W <= 0) return 0;
    return isb_edt_workspace_bytes(H, W) + isb_align((size_t)H * W);
}

extern "C" int isb_edt_2d_indices(const uint8_t* sites, int H, int W, int32_t* index, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(sites && index && ws, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0, "bad sizes");
    ISB_REQUIRE(H <= 32768 && W <= 32768, "the squared distances of an image larger than 32768 x 32768 overflow int32");
    ISB_REQUIRE(ws_bytes >= isb_edt_index_workspace_bytes(H, W), "workspace too small");
    return edt_run<true>(sites, H, W, index, ws, ws_bytes, (cudaStream_t)stream);
}

extern "C" size_t isb_mask_compact_workspace_bytes(int H, int W)
{
    if (H <= 0 || W <= 0) return 0;
    return compact_workspace_bytes((long long)H * W);
}

extern "C" int isb_mask_compact_count(const uint8_t* mask, int H, int W, void* ws, size_t ws_bytes, long long* total, isb_stream_t stream)
{
    ISB_REQUIRE(mask && ws && total, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0, "bad sizes");
    ISB_REQUIRE(ws_bytes >= isb_mask_compact_workspace_bytes(H, W), "workspace too small");
    return compact_count(mask, (long long)H * W, ws, (cudaStream_t)stream, total);
}

extern "C" int isb_mask_compact_write(const uint8_t* mask, int H, int W, const double* values, const void* ws, size_t ws_bytes, int64_t* points,
                                      double* values_out, isb_stream_t stream)
{
    ISB_REQUIRE(mask && ws && points, "null pointer");
    ISB_REQUIRE(!values || values_out, "values need values_out");
    ISB_REQUIRE(H > 0 && W > 0, "bad sizes");
    ISB_REQUIRE(ws_bytes >= isb_mask_compact_workspace_bytes(H, W), "workspace too small");
    const long long n = (long long)H * W;
    const int nt = compact_tiles(n);
    const long long* tile_off = compact_tile_offsets(ws, n);
    k_compact_write<<<nt, CPT_THREADS, 0, (cudaStream_t)stream>>>(mask, n, W, values, tile_off, points, values_out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_relabel_gather(const int32_t* seg, long long npx, const int32_t* lut, int n_lut, int32_t* out, isb_stream_t stream)
{
    ISB_REQUIRE(seg && lut && out, "null pointer");
    ISB_REQUIRE(npx > 0 && n_lut > 0, "bad sizes");
    k_relabel<<<(unsigned)((npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(seg, npx, lut, n_lut, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
