// lm_texture.cu -- Leung-Malik texture descriptors: background subtraction + filter-bank contraction + statistics.
//
// Replaces imsegm/descriptors.py:1041-1106 compute_texture_desc_lm_img2d_clr:
//   :1078      img - gaussian_filter(img.astype(float), 150)      (sigma 150 on ALL THREE axes, mode reflect, 1201 taps)
//   :1085-1098 per battery: ndimage.convolve of every channel with every 33x33 kernel, max over orientations (:951-966),
//              clip at 1e6 (:1088), scale by log(1 + ||r||) / 0.03 / ||r|| over the whole [3,H,W] response (:1090-1094),
//              per-superpixel mean / std / energy (compute_image2d_color_statistic -> features_cython.pyx)
//
// (1) background: separable FP64 correlation; one kernel blurs along the image rows axis with coalesced column access
//     (a thread owns a column and 16 consecutive output rows, the 1201 weights slide through registers), the other axis
//     reuses it on a transposed copy; the channel axis (length 3, reflected 1201-tap kernel) folds into a 3x3 mix.
// (2) contraction: implicit GEMM  response[pixel, filter] = sum_taps patch[pixel, tap] * K[tap, filter]  on the TENSOR
//     cores: wgmma.mma_async with TF32 inputs and the 3xTF32 split (a_hi b_hi + a_hi b_lo + a_lo b_hi, FP32 accumulate in
//     registers), which keeps the result at f32 accuracy -- the reference rounds every response to f32 before its statistics
//     (descriptors.py:233).  Source rows and the pre-split weights arrive by TMA; the patch matrices are gathered into registers.
//     FLOPs: 3 channels x 76 kernels x 33^2 x 2 = 496 584 per pixel (x3 for the split).
// (3) epilogue, fused: max over the orientations of a battery (quad shuffles), clip, then sum r and sum r^2 per
//     (superpixel, battery, channel) and globally per battery -- the responses are never written to memory.  The
//     log-norm scale is applied to the sums afterwards (mean and std scale with a, energy with a^2).
// Tolerance against the float64 oracle: every clipped response r within 1e-5 of M = max |img - background| (per pixel,
// tests/test_gpu_lm_responses.py; worst measured 2.2e-6 on an H100 80GB HBM3 at 700 W), so the features within 2e-4 of the battery
// response scale (tests/test_gpu_texture.py).
#include "common.cuh"
#include "wgmma.cuh"

namespace {

// ---------------------------------------------------------------- (1) background ----------------------------------------------------

constexpr int VB_R = 32;      // output rows per thread
constexpr int VB_T = 128;     // threads (columns) per CTA

__global__ void __launch_bounds__(256) k_lm_to_planar(const void* __restrict__ img, int dtype, size_t npx, double* __restrict__ out)
{
    size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npx) return;
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c * npx + p] = load_as_f64(img, dtype, 3 * p + c);
}

// blur along axis 0 of [planes][n0][n1] (n1 contiguous).  wfull: 2*radius+1 weights (symmetric), in global memory.
// A thread owns one column and R consecutive output rows.  Input rows are taken R at a time: the 2R - 1 weights such a block needs
// (output row r takes input row t with w[d + t - r]) sit in REGISTERS and slide by R per block -- R weight loads for R^2 FP64 FMAs.
// Every block of R output rows reads its own 2 radius + R input rows, so the L2 -> SM traffic is (2 radius / R + 1) x the image:
// R = 32 instead of 16 halves what turned out to be the bound of this kernel (3.2 TB/s of L2 reads at R = 16).
template <int R, bool FAST_REFLECT>
__global__ void __launch_bounds__(VB_T) k_lm_vblur(const double* __restrict__ in, int n0, int n1, const double* __restrict__ wfull, int radius,
                                                   double* __restrict__ out)
{
    // padded weights: s_w[d + radius + 3R] = w[d] for |d| <= radius, 0 for the 3R entries on either side (the last refill of the
    // register window reads up to 3R - 2 past the radius)
    extern __shared__ double s_w[];
    const int pad = radius + 3 * R, wn = 2 * pad + 1;
    for (int i = threadIdx.x; i < wn; i += VB_T) {
        int d = i - pad;
        s_w[i] = (d >= -radius && d <= radius) ? wfull[d + radius] : 0.0;
    }
    __syncthreads();
    const int x = blockIdx.x * VB_T + threadIdx.x;
    const int y0 = blockIdx.y * R;
    const size_t plane = (size_t)blockIdx.z * n0 * n1;
    if (x >= n1) return;
    double acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.0;
    // input rows i = y0 - radius .. y0 + R - 1 + radius (rounded up to whole blocks: the extra rows meet zero weights);
    // output row y0 + r uses weight w[i - (y0 + r)]
    const int n_blocks = (2 * radius + R + R - 1) / R;
    const double* wc = s_w + pad; // wc[d]
    double w[2 * R - 1];          // w[j] = wc[db - (R - 1) + j], db = offset of the block's first input row from output row y0
    int db = -radius;
#pragma unroll
    for (int j = 0; j < 2 * R - 1; ++j) w[j] = wc[db - (R - 1) + j];
    const double* col = in + plane + x;
    for (int blk = 0; blk < n_blocks; ++blk, db += R) {
#pragma unroll
        for (int t = 0; t < R; ++t) {
            int i = y0 + db + t;
            // one reflection is enough when radius + 2R <= n0 (FAST_REFLECT); the general form handles images smaller than the kernel
            if (FAST_REFLECT) i = i < 0 ? -1 - i : (i >= n0 ? 2 * n0 - 1 - i : i);
            else i = reflect_index(i, n0);
            const double v = col[(size_t)i * n1];
#pragma unroll
            for (int r = 0; r < R; ++r) acc[r] = fma(w[R - 1 + t - r], v, acc[r]);
        }
#pragma unroll
        for (int j = 0; j < R - 1; ++j) w[j] = w[j + R];
#pragma unroll
        for (int j = 0; j < R; ++j) w[R - 1 + j] = wc[db + R + j];
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
        if (y0 + r < n0) out[plane + (size_t)(y0 + r) * n1 + x] = acc[r];
}

static int launch_vblur(const double* in, int n0, int n1, const double* w, int radius, double* out, cudaStream_t st)
{
    const size_t smem = sizeof(double) * (2 * (size_t)(radius + 3 * VB_R) + 1);
    ISB_REQUIRE(smem <= 200 * 1024, "background radius too large");
    const dim3 grid((n1 + VB_T - 1) / VB_T, (n0 + VB_R - 1) / VB_R, 3);
    if (radius + 2 * VB_R <= n0) {
        ISB_CUDA_CHECK(cudaFuncSetAttribute(k_lm_vblur<VB_R, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_lm_vblur<VB_R, true><<<grid, VB_T, smem, st>>>(in, n0, n1, w, radius, out);
    } else {
        ISB_CUDA_CHECK(cudaFuncSetAttribute(k_lm_vblur<VB_R, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_lm_vblur<VB_R, false><<<grid, VB_T, smem, st>>>(in, n0, n1, w, radius, out);
    }
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// [planes][n0][n1] -> [planes][n1][n0]
__global__ void __launch_bounds__(256) k_lm_transpose(const double* __restrict__ in, int n0, int n1, double* __restrict__ out)
{
    __shared__ double tile[32][33];
    const size_t plane = (size_t)blockIdx.z * n0 * n1;
    const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (int j = ty; j < 32; j += 8)
        if (by + j < n0 && bx + tx < n1) tile[j][tx] = in[plane + (size_t)(by + j) * n1 + bx + tx];
    __syncthreads();
    for (int j = ty; j < 32; j += 8)
        if (bx + j < n1 && by + tx < n0) out[plane + (size_t)(bx + j) * n0 + by + tx] = tile[tx][j];
}

// out[c][y][x] = (float)(in[c][y][x] - sum_c' mix[c][c'] * blurT[c'][x][y])   (blurT is [3][W][H])
struct Mix3 { double m[9]; };
__global__ void __launch_bounds__(256) k_lm_mix_sub(const double* __restrict__ in, const double* __restrict__ blurT, int H, int W, Mix3 mix,
                                                    float* __restrict__ out)
{
    __shared__ double tile[3][32][33];
    const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const size_t npx = (size_t)H * W;
    for (int c = 0; c < 3; ++c)
        for (int j = ty; j < 32; j += 8)
            if (bx + j < W && by + tx < H) tile[c][j][tx] = blurT[c * npx + (size_t)(bx + j) * H + by + tx];
    __syncthreads();
    for (int j = ty; j < 32; j += 8) {
        const int y = by + j, x = bx + tx;
        if (y >= H || x >= W) continue;
        const double b0 = tile[0][tx][j], b1 = tile[1][tx][j], b2 = tile[2][tx][j];
        for (int c = 0; c < 3; ++c) {
            const double bl = mix.m[3 * c] * b0 + mix.m[3 * c + 1] * b1 + mix.m[3 * c + 2] * b2;
            out[c * npx + (size_t)y * W + x] = (float)(in[c * npx + (size_t)y * W + x] - bl);
        }
    }
}

// ---------------------------------------------------------------- (2)+(3) contraction + statistics ---------------------------------
//
// Implicit GEMM on the Hopper tensor cores: wgmma.mma_async kind tf32, FP32 accumulators in registers.
//   M = 128 consecutive pixels of one image row (two warpgroups of 64), N = the padded filter count (80 full bank / 48 short bank),
//   K = the 33 taps of one kernel row padded to 40 (5 instructions of K = 8), one such product per (output row, kernel row).
// A CTA (persistent, one per SM) owns tiles of TR = 3 output rows x 128 pixels of one channel.  For every SOURCE row s of the
// tile (3 + 32 of them) the patch matrix A_s[m][k] = row_s[x0 + m + k] is used for every output row r with kernel row
// dy = s - r:  acc[r] += A_s * B_dy^T.  A_s is a Toeplitz matrix, so it is never formed: every thread gathers its register
// fragments of A_s straight from the staged source row (four consecutive-ish floats per instruction, no bank conflicts).
// 3xTF32: image and weights are pre-split into a tf32 value and a tf32 remainder; acc += a_lo*b_hi + a_hi*b_lo + a_hi*b_hi
// (FP32 accumulate) keeps f32 accuracy -- the reference rounds every response to f32 before its statistics (descriptors.py:233).
// Warp roles (288 threads):
//   warps 0-7  two consumer warpgroups: A fragments from the staged row, 3 x 5 x 3 wgmma per source row, then the epilogue:
//              max over the orientations of a battery (quad shuffles), clip, run-length sums of r and r^2 along the row per
//              (battery, output row) -> atomics on the per-superpixel sums.  The responses are never written to memory.
//   warp 8     TMA producer: the split weights of kernel row dy (one cp.async.bulk per slice) into a ring of NBT slices, the
//              source rows (2-D tensor-map loads of the reflect-padded hi / lo planes) into a ring of NRAW slots
// A weight slice is loaded once per tile and serves the three output rows; the accumulators of a tile (3 x NPAD / 2 floats per
// thread) stay in registers until its epilogue.

constexpr int KW = 33;                    // kernel edge
constexpr int KRAD = 16;
constexpr int KPAD = 40;                  // taps of one kernel row, padded to a multiple of 8
constexpr int KC = KPAD / 4;              // 16-byte chunks along K
constexpr int TM = 128;                   // pixels per M tile (one image row segment)
constexpr int TR = 3;                     // output rows per CTA tile
constexpr int SROWS = TR + KW - 1;        // source rows per tile
constexpr int RAWW = TM + KPAD;           // floats of one staged source row
constexpr int RAW_PITCH = 768;            // bytes between the hi and the lo row of a raw slot (TMA destinations 128-byte aligned)
constexpr int NRAW = 4;                   // ring depth of the staged source rows
constexpr int LM_CONS = 256;              // consumer threads: two warpgroups
constexpr int LM_THREADS = LM_CONS + 32;     // + the producer warp

struct LmTcArgs {
    const float* w_tc;   // [KW][hi|lo][KC][NPAD/8][8][4]: the weights of every kernel row in operand layout
    const int* seg;      // [H][W]
    int H, W, tiles_x, tiles_y, Hp;
    int y_first, y_end;  // rows [y_first, y_end) of the slab are this call's: tiles start at y_first, rows >= y_end are masked
    int n_batt;
    double* S1;          // [nb][n_batt*3] sum r
    double* S2;          // [nb][n_batt*3] sum r^2
    double* G2;          // [n_batt] global sum r^2 over all pixels and channels
};

template <int NPAD> struct LmBank;
template <> struct LmBank<80> { static constexpr int GS = 8, NG = 8, NS = 12, NBATT = 20; };   // 4 sigmas x (edge, bar) x 8 orientations
template <> struct LmBank<48> { static constexpr int GS = 4, NG = 6, NS = 9, NBATT = 15; };    // 3 sigmas x (edge, bar) x 4 orientations

// battery of an accumulator column: oriented groups first (edge s0 | bar s0 | edge s1 | ...), then Gauss / LoG / LoG2 per sigma
template <int NPAD> __host__ __device__ constexpr int lm_batt_of_col(int col)
{
    using Bk = LmBank<NPAD>;
    if (col < Bk::GS * Bk::NG) return 5 * ((col / Bk::GS) / 2) + ((col / Bk::GS) % 2);
    return (col - Bk::GS * Bk::NG) < Bk::NS ? 5 * ((col - Bk::GS * Bk::NG) / 3) + 2 + (col - Bk::GS * Bk::NG) % 3 : -1;
}

// Shared memory: a ring of NBT weight slices, each [hi|lo][KC k-chunks][NPAD/8 filter groups][8 x 16 B] exactly as w_tc holds a kernel
// row (descriptor LBO = one k-chunk, SBO = 128 B), the source-row ring, the battery maxima of a tile and its labels.
template <int NPAD> struct LmTs {
    using Bk = LmBank<NPAD>;
    static constexpr int NBT = NPAD == 80 ? 5 : 8;                                   // weight slices in flight
    static constexpr int SLOTC = (NPAD / 8) * 128;                                   // bytes of one (half, k-chunk): NPAD filters x 4 taps
    static constexpr int B_SLICE = 2 * KC * SLOTC;                                   // bytes of one weight slice (value + remainder)
    static constexpr int TS = Bk::NBATT + 1;
    static constexpr int OFF_B = 0;
    static constexpr int OFF_RAW = OFF_B + NBT * B_SLICE;
    static constexpr int OFF_T = OFF_RAW + NRAW * 2 * RAW_PITCH;
    static constexpr int OFF_LAB = OFF_T + TR * TM * TS * 4;
    static constexpr int OFF_BAR = OFF_LAB + TR * TM * 4;
    static constexpr int N_BAR = 2 * NRAW + 2 * NBT;
    static constexpr int BYTES = OFF_BAR + N_BAR * 8;
    static_assert(NBT >= TR + 1, "the weight ring must hold the TR slices in use and one in flight");
    static_assert(OFF_RAW % 128 == 0, "TMA destinations are 128-byte aligned");
    static_assert((Bk::GS * Bk::NG) % 8 == 0 && 8 % Bk::GS == 0, "an 8-column accumulator group holds whole oriented batteries");
    static_assert(BYTES <= 227 * 1024, "shared memory budget");
};

// acc[r] += A_s * B_{s-r}^T for the output rows r = R_LO..R_HI, 3xTF32 (small terms first); slice dy of the tile is ring slot
// (jb_base + dy) % NBT, j0 = jb_base + s
template <int NPAD, int R_LO, int R_HI>
__device__ __forceinline__ void lm_issue(float (&acc)[TR][NPAD / 2], const uint32_t (&ah)[KPAD / 8][4], const uint32_t (&al)[KPAD / 8][4],
                                         uint32_t b_ring, uint32_t j0)
{
    using namespace wgmma;
    using Sm = LmTs<NPAD>;
    wg_fence();
#pragma unroll
    for (int r = R_LO; r <= R_HI; ++r) {
        const uint32_t b_hi = b_ring + ((j0 - r) % Sm::NBT) * Sm::B_SLICE, b_lo = b_hi + KC * Sm::SLOTC;
#pragma unroll
        for (int kk = 0; kk < KPAD / 8; ++kk) {
            const uint64_t bh = smem_desc(b_hi + kk * 2 * Sm::SLOTC, Sm::SLOTC, 128);
            const uint64_t bl = smem_desc(b_lo + kk * 2 * Sm::SLOTC, Sm::SLOTC, 128);
            mma_tf32_rs(acc[r], al[kk], bh, 1);
            mma_tf32_rs(acc[r], ah[kk], bl, 1);
            mma_tf32_rs(acc[r], ah[kk], bh, 1);
        }
    }
    wg_commit();
    wg_wait<0>();
}

// np.max over the orientations and `resp[resp > 1e6] = 1e6` (descriptors.py:1088) both keep a NaN response, so that a NaN or infinite
// pixel makes the battery's norm NaN and k_lm_finalize writes zeros, as np.nan_to_num does on the reference's NaN features.  fmaxf and
// fminf would return the other operand instead.
__device__ __forceinline__ float max_keep_nan(float a, float b)
{
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

__device__ __forceinline__ float clip_response(float v) { return v > 1.e6f ? 1.e6f : v; }   // MAX_SIGNAL_RESPONSE

template <int NPAD>
__global__ void __launch_bounds__(LM_THREADS, 1) k_lm_conv_wg(const __grid_constant__ CUtensorMap tmap, LmTcArgs a)
{
    using namespace wgmma;
    using Sm = LmTs<NPAD>;
    using Bk = LmBank<NPAD>;
    constexpr int NBT = Sm::NBT;
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t sbase = smem_u32(smem);
    const uint32_t bar0 = sbase + Sm::OFF_BAR;
    auto raw_full = [&](uint32_t i) { return bar0 + 8u * i; };
    auto raw_empty = [&](uint32_t i) { return bar0 + 8u * (NRAW + i); };
    auto b_full = [&](uint32_t i) { return bar0 + 8u * (2 * NRAW + i); };
    auto b_empty = [&](uint32_t i) { return bar0 + 8u * (2 * NRAW + NBT + i); };

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int i = 0; i < NRAW; ++i) { mbar_init(raw_full(i), 1); mbar_init(raw_empty(i), LM_CONS / 32); }
        for (int i = 0; i < NBT; ++i) { mbar_init(b_full(i), 1); mbar_init(b_empty(i), LM_CONS / 32); }
        fence_mbar_init();
        prefetch_tmap(&tmap);
    }
    __syncthreads();

    const int tiles_per_ch = a.tiles_x * a.tiles_y;
    const int n_tiles = 3 * tiles_per_ch;

    if (warp == LM_CONS / 32) {
        // ------------------------------------------------------------ TMA producer ------------------------------------------------
        if (lane == 0) {
            uint32_t jr = 0, jb = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
                const int ch = t / tiles_per_ch, rem = t - ch * tiles_per_ch;
                const int ty = rem / a.tiles_x, tx = rem - ty * a.tiles_x;
                const int x0 = tx * TM, y0 = a.y_first + ty * TR;
                for (int s = 0; s < SROWS; ++s) {
                    if (s < KW) {
                        // kernel row s: value and remainder in one piece
                        const uint32_t slot = jb % NBT;
                        mbar_wait(b_empty(slot), ((jb / NBT) & 1) ^ 1);
                        mbar_arrive_expect_tx(b_full(slot), Sm::B_SLICE);
                        bulk_g2s(sbase + Sm::OFF_B + slot * Sm::B_SLICE, a.w_tc + (size_t)s * (Sm::B_SLICE / 4), Sm::B_SLICE, b_full(slot));
                        ++jb;
                    }
                    const uint32_t slot = jr % NRAW;
                    mbar_wait(raw_empty(slot), ((jr / NRAW) & 1) ^ 1);
                    mbar_arrive_expect_tx(raw_full(slot), 2 * RAWW * 4);
                    const uint32_t dst = sbase + Sm::OFF_RAW + slot * 2 * RAW_PITCH;
                    tma_load_2d(dst, &tmap, x0, ch * a.Hp + y0 + s, raw_full(slot));
                    tma_load_2d(dst + RAW_PITCH, &tmap, x0, (3 + ch) * a.Hp + y0 + s, raw_full(slot));
                    ++jr;
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers --------------------------------------------------
    const int e = threadIdx.x;                         // 0..255
    const int tq = lane & 3;
    const int m0 = 16 * warp + (lane >> 2);            // pixel of accumulator rows i % 4 < 2; m0 + 8 for the others (warp 4.. = rows 64..)
    float* T = (float*)(smem + Sm::OFF_T);
    int* s_lab = (int*)(smem + Sm::OFF_LAB);
    const bool walker = e < 2 * TR * Bk::NBATT;
    const int p = e >> 1, half = e & 1;
    const int wr = p / Bk::NBATT, wb = p - wr * Bk::NBATT;
    double g2 = 0.0;
    uint32_t jr = 0, jb_base = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, jb_base += KW) {
        const int ch = t / tiles_per_ch, rem = t - ch * tiles_per_ch;
        const int ty = rem / a.tiles_x, tx = rem - ty * a.tiles_x;
        const int x0 = tx * TM, y0 = a.y_first + ty * TR;
        float acc[TR][NPAD / 2];
#pragma unroll
        for (int r = 0; r < TR; ++r)
#pragma unroll
            for (int i = 0; i < NPAD / 2; ++i) acc[r][i] = 0.f;
        for (int s = 0; s < SROWS; ++s, ++jr) {
            if (s < KW) { const uint32_t jb = jb_base + s; mbar_wait(b_full(jb % NBT), (jb / NBT) & 1); }
            const uint32_t rs = jr % NRAW;
            mbar_wait(raw_full(rs), (jr / NRAW) & 1);
            // A fragments: rows m0 / m0 + 8, taps tq / tq + 4 of every K = 8 step -> row_s[m + k]
            const float* hi = (const float*)(smem + Sm::OFF_RAW + rs * 2 * RAW_PITCH) + m0 + tq;
            const float* lo = hi + RAW_PITCH / 4;
            uint32_t ah[KPAD / 8][4], al[KPAD / 8][4];
#pragma unroll
            for (int kk = 0; kk < KPAD / 8; ++kk) {
                ah[kk][0] = __float_as_uint(hi[8 * kk]); ah[kk][1] = __float_as_uint(hi[8 * kk + 8]);
                ah[kk][2] = __float_as_uint(hi[8 * kk + 4]); ah[kk][3] = __float_as_uint(hi[8 * kk + 12]);
                al[kk][0] = __float_as_uint(lo[8 * kk]); al[kk][1] = __float_as_uint(lo[8 * kk + 8]);
                al[kk][2] = __float_as_uint(lo[8 * kk + 4]); al[kk][3] = __float_as_uint(lo[8 * kk + 12]);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(raw_empty(rs));
            // output rows R_LO..R_HI take this source row with kernel row dy = s - r; the range is a compile-time property of the
            // call so that every wgmma of the warpgroup sits on one straight path
            const uint32_t b0 = sbase + Sm::OFF_B;
            const uint32_t j0 = jb_base + s;
            if (s == 0) lm_issue<NPAD, 0, 0>(acc, ah, al, b0, j0);
            else if (s < TR - 1) lm_issue<NPAD, 0, TR - 2>(acc, ah, al, b0, j0);
            else if (s < KW) lm_issue<NPAD, 0, TR - 1>(acc, ah, al, b0, j0);
            else if (s < SROWS - 1) lm_issue<NPAD, 1, TR - 1>(acc, ah, al, b0, j0);
            else lm_issue<NPAD, TR - 1, TR - 1>(acc, ah, al, b0, j0);
            if (s >= TR - 1) {                                 // kernel row s - (TR-1) had its last use
                __syncwarp();
                if (lane == 0) mbar_arrive(b_empty((jb_base + s - (TR - 1)) % NBT));
            }
        }
        // ------------------------------------------------------------ epilogue ------------------------------------------------------
        for (int i = e; i < TR * TM; i += LM_CONS) {
            const int y = y0 + i / TM, x = x0 + i % TM;
            s_lab[i] = (y < a.y_end && x < a.W) ? a.seg[(size_t)y * a.W + x] : -1;
        }
#pragma unroll
        for (int r = 0; r < TR; ++r) {
#pragma unroll
            for (int j = 0; j < NPAD / 8; ++j) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float* row = T + (size_t)(r * TM + m0 + 8 * h) * Sm::TS;
                    const float v0 = acc[r][4 * j + 2 * h], v1 = acc[r][4 * j + 2 * h + 1];
                    const int c0 = 8 * j + 2 * tq;
                    if (8 * j < Bk::GS * Bk::NG) {
                        // an oriented battery spans GS adjacent columns = GS / 2 threads of the quad
                        float v = max_keep_nan(v0, v1);
                        v = max_keep_nan(v, __shfl_xor_sync(0xffffffffu, v, 1));
                        if (Bk::GS == 8) v = max_keep_nan(v, __shfl_xor_sync(0xffffffffu, v, 2));
                        if (tq % (Bk::GS / 2) == 0) row[lm_batt_of_col<NPAD>(c0)] = clip_response(v);
                    } else {
                        const int b0 = lm_batt_of_col<NPAD>(c0), b1 = lm_batt_of_col<NPAD>(c0 + 1);
                        if (b0 >= 0) row[b0] = clip_response(v0);
                        if (b1 >= 0) row[b1] = clip_response(v1);
                    }
                }
            }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(LM_CONS) : "memory");
        if (walker) {
            // one (output row, battery) pair and half a row per thread: run-length sums along x, flushed when the label changes
            const size_t fstride = (size_t)a.n_batt * 3;
            double s1 = 0.0, s2 = 0.0;
            int cur = -1;
            const int* lab = s_lab + wr * TM + half * (TM / 2);
            const float* tv = T + (size_t)(wr * TM + half * (TM / 2)) * Sm::TS + wb;
            for (int i = 0; i < TM / 2; ++i) {
                const int lb = lab[i];
                if (lb != cur) {
                    if (cur >= 0) {
                        atomicAdd(&a.S1[(size_t)cur * fstride + wb * 3 + ch], s1);
                        atomicAdd(&a.S2[(size_t)cur * fstride + wb * 3 + ch], s2);
                        g2 += s2;
                    }
                    cur = lb; s1 = 0.0; s2 = 0.0;
                }
                if (lb >= 0) { const double v = (double)tv[(size_t)i * Sm::TS]; s1 += v; s2 += v * v; }
            }
            if (cur >= 0) {
                atomicAdd(&a.S1[(size_t)cur * fstride + wb * 3 + ch], s1);
                atomicAdd(&a.S2[(size_t)cur * fstride + wb * 3 + ch], s2);
                g2 += s2;
            }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(LM_CONS) : "memory");
    }
    if (walker && g2 != 0.0) atomicAdd(&a.G2[wb], g2);
}

// reflect-padded, tf32-split planes for the tensor-map loads: P[c][yp][xp] = split(img[c][reflect(yp - 16)][reflect(xp - 16)]);
// rows [0, 3 Hp) hold the tf32 values, rows [3 Hp, 6 Hp) the tf32 remainders
__global__ void __launch_bounds__(256) k_lm_pad_split(const float* __restrict__ img, int H, int W, int Hp, int Wp, float* __restrict__ P)
{
    const int xp = blockIdx.x * blockDim.x + threadIdx.x, yp = blockIdx.y, c = blockIdx.z;
    if (xp >= Wp) return;
    const float v = img[(size_t)c * H * W + (size_t)reflect_index(yp - KRAD, H) * W + reflect_index(xp - KRAD, W)];
    unsigned hb, lb;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hb) : "f"(v));
    const float hi = __uint_as_float(hb);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lb) : "f"(v - hi));
    P[((size_t)c * Hp + yp) * Wp + xp] = hi;
    P[((size_t)(3 + c) * Hp + yp) * Wp + xp] = __uint_as_float(lb);
}

__device__ __forceinline__ double tidy(double v)
{
    if (isnan(v)) return 0.0;
    return v == 0.0 ? 0.0 : v;
}

// features = statistics of the scaled responses: a = log(1 + ||r||) / 0.03 / ||r|| per battery
__global__ void k_lm_finalize(int nb, int n_batt, int flags, const double* __restrict__ S1, const double* __restrict__ S2,
                              const double* __restrict__ G2, const int* __restrict__ counts, double* feat, int ld, int col0)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nb * n_batt) return;
    const int k = i / n_batt, b = i - k * n_batt;
    const double norm = sqrt(G2[b]);
    const double al = (norm == 0.0 || isinf(norm)) ? 0.0 : (log(1.0 + norm) / 0.03) / norm;
    const int nfl = ((flags & 1) ? 1 : 0) + ((flags & 2) ? 1 : 0) + ((flags & 4) ? 1 : 0);
    const double n = (double)counts[k];
    double* row = feat + (size_t)k * ld + col0 + (size_t)b * 3 * nfl;
    for (int c = 0; c < 3; ++c) {
        const double s1 = S1[(size_t)k * n_batt * 3 + b * 3 + c], s2 = S2[(size_t)k * n_batt * 3 + b * 3 + c];
        double mean = 0, en = 0, sd = 0;
        if (n > 0) {
            mean = al * s1 / n;
            en = al * al * s2 / n;
            double var = en - mean * mean;
            sd = var > 0 ? sqrt(var) : 0.0;
        }
        int col = 0;
        if (flags & 1) { row[col * 3 + c] = tidy(mean); ++col; }
        if (flags & 2) { row[col * 3 + c] = tidy(sd); ++col; }
        if (flags & 4) { row[col * 3 + c] = tidy(en); ++col; }
    }
}

__global__ void k_lm_counts(const int* __restrict__ seg, size_t npx, int* counts)
{
    // neighbouring pixels mostly share a label: one atomic per (warp, label) instead of one per pixel
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = p < npx;
    const unsigned act = __ballot_sync(0xffffffffu, in);
    if (!in) return;
    const int lb = seg[p];
    const unsigned grp = __match_any_sync(act, lb);
    if ((int)(threadIdx.x & 31) == __ffs(grp) - 1) atomicAdd(&counts[lb], __popc(grp));
}

struct LmWs { double* p0; double* p1; double* p2; float* imgf; float* planes; double* acc; int* counts; };

// accumulators of one image: S1 [nb][n_batt*3] | S2 [nb][n_batt*3] | G2 [32], one block so that the banded path sums it with one all_reduce
static size_t lm_acc_doubles(int nb, int n_batt) { return 2 * (size_t)nb * n_batt * 3 + 32; }

struct LmDims { int tiles_x, Hp, Wp; };
static LmDims lm_dims(int H, int W)
{
    LmDims d;
    d.tiles_x = (W + TM - 1) / TM;
    d.Hp = ((H + TR - 1) / TR + 1) * TR + KW - 1;   // every source row a tile asks for exists, wherever the first tile row starts
    d.Wp = d.tiles_x * TM + KPAD;                   // a multiple of 4 floats: tensor-map row pitch is a multiple of 16 bytes
    return d;
}

static size_t carve_lm(LmWs& w, void* ws, size_t bytes, int H, int W, int nb, int n_batt)
{
    WsCarver c(ws, bytes);
    const size_t n = 3 * (size_t)H * W;
    const LmDims d = lm_dims(H, W);
    w.p0 = c.take<double>(n); w.p1 = c.take<double>(n); w.p2 = c.take<double>(n);
    w.imgf = c.take<float>(n);
    w.planes = c.take<float>(6 * (size_t)d.Hp * d.Wp);
    w.acc = c.take<double>(lm_acc_doubles(nb, n_batt));
    w.counts = c.take<int>(nb);
    return isb_align(c.off);
}

template <int NPAD>
static int launch_lm_conv(const CUtensorMap& tmap, const LmTcArgs& a, int n_tiles, cudaStream_t st)
{
    int dev = 0, sms = 0;
    ISB_CUDA_CHECK(cudaGetDevice(&dev));
    ISB_CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int grid = n_tiles < sms ? n_tiles : sms;   // persistent: one CTA per SM, tiles round-robin
    ISB_CUDA_CHECK(cudaFuncSetAttribute(k_lm_conv_wg<NPAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, LmTs<NPAD>::BYTES));
    k_lm_conv_wg<NPAD><<<grid, LM_THREADS, LmTs<NPAD>::BYTES, st>>>(tmap, a);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// background subtraction + contraction over the slab img [H][W][3]; the sums of the rows [y_first, y_end) are ADDED to acc / counts
static int lm_accumulate(const void* img, int dtype, const int32_t* seg, int H, int W, int y_first, int y_end, int nb, const double* bg_weights,
                         int bg_radius, const double* chmix_host, const float* w_tc, int orient, int n_batt, const LmWs& w, double* acc,
                         int* counts, cudaStream_t st)
{
    const size_t npx = (size_t)H * W;
    k_lm_to_planar<<<(unsigned)((npx + 255) / 256), 256, 0, st>>>(img, dtype, npx, w.p0);
    ISB_LAUNCH_CHECK();
    Mix3 mix;
    for (int i = 0; i < 9; ++i) mix.m[i] = chmix_host[i];
    if (bg_radius > 0) {
        // axis 0 (rows): p0 [3][H][W] -> p1
        if (int rc = launch_vblur(w.p0, H, W, bg_weights, bg_radius, w.p1, st)) return rc;
        // axis 1 (cols): transpose, blur along the (new) rows axis; the result stays transposed [3][W][H]
        k_lm_transpose<<<dim3((W + 31) / 32, (H + 31) / 32, 3), 256, 0, st>>>(w.p1, H, W, w.p2);
        ISB_LAUNCH_CHECK();
        if (int rc = launch_vblur(w.p2, W, H, bg_weights, bg_radius, w.p1, st)) return rc;
    } else {
        ISB_CUDA_CHECK(cudaMemsetAsync(w.p1, 0, sizeof(double) * 3 * npx, st));
    }
    // axis 2 (channels) folded into the 3x3 mix; subtract; to f32 planar
    k_lm_mix_sub<<<dim3((W + 31) / 32, (H + 31) / 32), 256, 0, st>>>(w.p0, w.p1, H, W, mix, w.imgf);
    ISB_LAUNCH_CHECK();
    // reflect-padded tf32 value / remainder planes, and the tensor map the contraction's TMA loads read them through
    const LmDims d = lm_dims(H, W);
    k_lm_pad_split<<<dim3((d.Wp + 255) / 256, d.Hp, 3), 256, 0, st>>>(w.imgf, H, W, d.Hp, d.Wp, w.planes);
    ISB_LAUNCH_CHECK();
    wgmma::EncodeTiledFn encode = wgmma::encode_tiled_fn();
    if (!encode) { isb_set_error("cuTensorMapEncodeTiled is not available from this driver"); return ISB_ERR_UNSUPPORTED; }
    CUtensorMap tmap;
    {
        const cuuint64_t gdim[2] = { (cuuint64_t)d.Wp, (cuuint64_t)6 * d.Hp };
        const cuuint64_t gstride[1] = { (cuuint64_t)d.Wp * sizeof(float) };
        const cuuint32_t box[2] = { (cuuint32_t)RAWW, 1 };
        const cuuint32_t estr[2] = { 1, 1 };
        const CUresult r = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)w.planes, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { isb_set_error("cuTensorMapEncodeTiled failed with CUresult %d", (int)r); return ISB_ERR_CUDA; }
    }
    const size_t nown = (size_t)(y_end - y_first) * W;
    k_lm_counts<<<(unsigned)((nown + 255) / 256), 256, 0, st>>>(seg + (size_t)y_first * W, nown, counts);
    ISB_LAUNCH_CHECK();
    LmTcArgs a;
    a.w_tc = w_tc; a.seg = seg; a.H = H; a.W = W; a.tiles_x = d.tiles_x; a.tiles_y = (y_end - y_first + TR - 1) / TR; a.Hp = d.Hp; a.n_batt = n_batt;
    a.y_first = y_first; a.y_end = y_end;
    a.S1 = acc; a.S2 = acc + (size_t)nb * n_batt * 3; a.G2 = acc + 2 * (size_t)nb * n_batt * 3;
    const int n_tiles = 3 * a.tiles_x * a.tiles_y;
    return orient == 8 ? launch_lm_conv<80>(tmap, a, n_tiles, st) : launch_lm_conv<48>(tmap, a, n_tiles, st);
}

static bool lm_bank_ok(int NP, int orient, int n_batt)
{
    return (orient == 8 && NP == 80 && n_batt == 20) || (orient == 4 && NP == 48 && n_batt == 15);
}

} // namespace

extern "C" size_t isb_lm_workspace_bytes(int H, int W, int nb, int n_batt)
{
    LmWs w;
    return carve_lm(w, nullptr, 0, H, W, nb, n_batt);
}

extern "C" size_t isb_lm_acc_doubles(int nb, int n_batt) { return lm_acc_doubles(nb, n_batt); }

extern "C" int isb_lm_texture(const void* img, int dtype, const int32_t* seg, int H, int W, int nb, const double* bg_weights, int bg_radius,
                              const double* chmix_host, const float* w_tc, int NP, int orient, int n_batt, int flags,
                              double* feat, int ld, int col0, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(img && seg && w_tc && feat && ws && chmix_host, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && nb > 0, "bad sizes");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    ISB_REQUIRE(lm_bank_ok(NP, orient, n_batt),
                "filter bank layout must be the full (8 orientations, 80 padded filters, 20 batteries) or the short one (4, 48, 15)");
    ISB_REQUIRE(bg_radius >= 0 && (bg_radius == 0 || bg_weights), "background weights missing");
    LmWs w;
    size_t need = carve_lm(w, ws, ws_bytes, H, W, nb, n_batt);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_LM, st);
    ISB_CUDA_CHECK(cudaMemsetAsync(w.acc, 0, sizeof(double) * lm_acc_doubles(nb, n_batt), st));
    ISB_CUDA_CHECK(cudaMemsetAsync(w.counts, 0, sizeof(int) * (size_t)nb, st));
    if (int rc = lm_accumulate(img, dtype, seg, H, W, 0, H, nb, bg_weights, bg_radius, chmix_host, w_tc, orient, n_batt, w, w.acc, w.counts, st))
        return rc;
    const size_t n3 = (size_t)nb * n_batt * 3;
    k_lm_finalize<<<(nb * n_batt + 255) / 256, 256, 0, st>>>(nb, n_batt, flags, w.acc, w.acc + n3, w.acc + 2 * n3, w.counts, feat, ld, col0);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

// Row-band mode (one image over several GPUs): the slab img [slab_rows][W][3] holds the rows this band owns, [y_first, y_end) in slab
// coordinates, plus a halo of the background radius + 16 rows on every side that is not an image border (at an image border the slab
// ends and the reflection there is the image's own).  The sums of the owned rows are ADDED to acc (isb_lm_acc_doubles doubles, zeroed
// by the caller) and counts [nb]; after the bands' accumulators are summed, isb_lm_texture_finish forms the features.
extern "C" int isb_lm_texture_accumulate(const void* img, int dtype, const int32_t* seg, int slab_rows, int W, int y_first, int y_end, int nb,
                                         const double* bg_weights, int bg_radius, const double* chmix_host, const float* w_tc, int NP,
                                         int orient, int n_batt, double* acc, int32_t* counts, void* ws, size_t ws_bytes, isb_stream_t stream)
{
    ISB_REQUIRE(img && seg && w_tc && acc && counts && ws && chmix_host, "null pointer");
    ISB_REQUIRE(slab_rows > 0 && W > 0 && nb > 0 && y_first >= 0 && y_first < y_end && y_end <= slab_rows, "bad sizes");
    ISB_REQUIRE(dtype >= ISB_U8 && dtype <= ISB_F64, "bad dtype");
    ISB_REQUIRE(lm_bank_ok(NP, orient, n_batt),
                "filter bank layout must be the full (8 orientations, 80 padded filters, 20 batteries) or the short one (4, 48, 15)");
    ISB_REQUIRE(bg_radius >= 0 && (bg_radius == 0 || bg_weights), "background weights missing");
    LmWs w;
    size_t need = carve_lm(w, ws, ws_bytes, slab_rows, W, nb, n_batt);
    ISB_REQUIRE(need <= ws_bytes, "workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope prof(ISB_PROF_LM, st);
    return lm_accumulate(img, dtype, seg, slab_rows, W, y_first, y_end, nb, bg_weights, bg_radius, chmix_host, w_tc, orient, n_batt, w, acc, counts, st);
}

extern "C" int isb_lm_texture_finish(int nb, int n_batt, int flags, const double* acc, const int32_t* counts, double* feat, int ld, int col0,
                                     isb_stream_t stream)
{
    ISB_REQUIRE(acc && counts && feat, "null pointer");
    ISB_REQUIRE(nb > 0 && (n_batt == 20 || n_batt == 15), "bad sizes");
    const size_t n3 = (size_t)nb * n_batt * 3;
    k_lm_finalize<<<(nb * n_batt + 255) / 256, 256, 0, (cudaStream_t)stream>>>(nb, n_batt, flags, acc, acc + n3, acc + 2 * n3, counts, feat, ld, col0);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
