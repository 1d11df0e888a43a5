/*
 * imsegm_b200.h -- C-ABI of the H100-native (sm_90a) SLIC -> descriptors -> GraphCut hot path of Borda/pyImSegm.
 *
 * Every entry point takes plain DEVICE pointers (unless a parameter says "host"), sizes and a CUDA stream
 * (cudaStream_t passed as void*), returns 0 on success or a negative isb_status, never allocates what it
 * returns and never throws.  isb_last_error() gives the message of the last failure on the calling thread.
 * The caller owns all buffers; `ws` is scratch the caller sizes with the matching *_workspace_bytes().
 * All launches are asynchronous on `stream` unless a parameter is documented as a host output.
 *
 * Each declaration names the reference interface it replaces (file:line under the reference repository).
 */
#ifndef IMSEGM_B200_H
#define IMSEGM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* isb_stream_t; /* cudaStream_t */

enum isb_status {
    ISB_OK = 0,
    ISB_ERR_ARG = -1,      /* bad argument (null pointer, non-positive size, unsupported dtype...) */
    ISB_ERR_CUDA = -2,     /* a CUDA runtime call failed; see isb_last_error() */
    ISB_ERR_CAPACITY = -3, /* a caller-sized table was too small (edge table, candidate list); retry larger */
    ISB_ERR_UNSUPPORTED = -4
};

/* ISB_I8 .. ISB_BOOL are taken by the label maps of isb_contingency_count / _write only */
enum isb_dtype { ISB_U8 = 0, ISB_U16 = 1, ISB_F32 = 2, ISB_F64 = 3, ISB_I8 = 4, ISB_I16 = 5, ISB_I32 = 6, ISB_U32 = 7, ISB_I64 = 8, ISB_BOOL = 9 };

const char* isb_last_error(void);
int isb_abi_version(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches) */
long long isb_launch_count(void);
/* a caller that replays a captured CUDA graph of this library's kernels reports the kernels of one replay here, so that
 * isb_launch_count() keeps counting kernels, not graph launches */
int isb_note_graph_replay(long long n_kernels);
/* per-stage device timers: CUDA events recorded on the launching stream around each stage's kernels while enabled.
 * isb_profile_collect() synchronises the recorded events and returns, per stage id, the summed milliseconds and
 * the number of timed launches (arrays of isb_profile_stage_count() entries); it clears the record list. */
int isb_profile_enable(int on);
int isb_profile_stage_count(void);
const char* isb_profile_stage_name(int id);
int isb_profile_collect(double* ms_out /* host */, long long* count_out /* host */);

/* ------------------------------------------------------------------------------------------------------------------
 * (i) SLIC -- replaces skimage.segmentation.slic as called from imsegm/superpixels.py:61-63
 *     slic(img f64[H,W,3] in [0,1], n_segments, compactness, sigma=1, enforce_connectivity=True, slic_zero)
 * ------------------------------------------------------------------------------------------------------------------ */

/* min-max rescale to [0,1] (imsegm/superpixels.py:53-54; in float32 for an ISB_F32 image, as numpy computes it, in f64
 * otherwise), gaussian pre-blur (scipy.ndimage semantics: symmetric
 * 1-D correlate, mode reflect, depth(len 1) -> rows -> cols), rgb2lab, multiply by ratio = 1/compactness.
 *   img        : [H,W,C] interleaved, C in {1,3} (gray is replicated, superpixels.py:50-51), dtype = isb_dtype
 *   w_half     : HOST pointer, radius+1 doubles, w_half[0] = centre tap (radius <= 8; radius 0 = no blur)
 *   lab_planar : out, [3,H,W] f64
 *   minmax_out : out, 4 doubles (device) -- [0] min and [1] max of the raw image ([2..3] scratch); max == min, or a NaN
 *                sample (both extrema are then NaN), makes the result NaN
 *   rescale    : 1 = apply the reference wrapper's min-max rescale when (min != 0 or max != 1); 0 = never;
 *                2 = as 1 with the extrema the caller left in minmax_out[0..1] (row-band mode: the extrema of the whole
 *                image, merged by a collective from isb_image_minmax of every band) */
int isb_slic_prepare(const void* img, int dtype, int H, int W, int C, const double* w_half, int radius, double ratio,
                     int rescale, double* lab_planar, double* minmax_out /* room for 4 doubles */, isb_stream_t stream);

/* minimum and maximum of n samples -> minmax_out[0..1]; [2..3] scratch.  numpy's rule: when any sample is NaN, both are NaN */
int isb_image_minmax(const void* img, int dtype, long long n, double* minmax_out /* room for 4 doubles */, isb_stream_t stream);

size_t isb_slic_kmeans_workspace_bytes(int H, int W, int n_seeds, int step_y, int step_x);

/* k-means sweeps of _slic_cython: window +-2*step about each centroid, lowest index wins ties, centroid = raster
 * order sequential double sums / count.  Bit-exact with oracle/slic_oracle.c by construction.
 *   seeds_yx  : [n_seeds,2] f64 (row, col) regular grid (device)
 *   labels    : out [H,W] i32;  centroids : optional out [n_seeds,5] f64 (y,x,L,a,b) */
int isb_slic_kmeans(const double* lab_planar, int H, int W, const double* seeds_yx, int n_seeds, int step_y, int step_x,
                    double step, int max_iter, int slic_zero, int32_t* labels, double* centroids, void* ws, size_t ws_bytes,
                    isb_stream_t stream);

/* Test hooks of the sweeps' per-tile candidate lists.  isb_slic_set_tile_cap(cap > 0) caps the list of every tile at cap
 * records for workspaces sized afterwards (0 restores the default sizing) and returns the previous cap; a tile whose list
 * overflows is assigned by scanning every cluster, with the same result.  isb_slic_full_scan_tiles counts those tile
 * assignments on the current device since the library was loaded. */
int isb_slic_set_tile_cap(int cap);
long long isb_slic_full_scan_tiles(void);

/* Row-band form of the sweeps: one image taller than a GPU wants to hold (BASELINE config 5, SURVEY.md section 8e) is cut into
 * row bands, one per GPU.  The cluster state (centres, windows) is replicated in every band's workspace and lives in
 * the coordinates of the whole image; a band holds pixel memory for its owned rows plus a halo of >= 2*step_y rows on either
 * side, assigns every row of that slab and sums the clusters whose centre row it owns (all their members are inside the slab;
 * a member further away -- an orphan that no window covers -- is counted in xchg[6 n_seeds] and the caller must then fall back
 * to one GPU).  Per sweep:
 *     isb_slic_band_assign -> isb_slic_band_update(xchg) -> [sum xchg as int64 over the bands] -> isb_slic_band_import(xchg)
 *     -> (SLICO: [max of maxdc_xchg as int64/uint64 over the bands]) -> isb_slic_band_finalize
 * xchg is [6*n_seeds + 1] int64: per cluster the bit patterns of (cy, cx, c0, c1, c2) and a state word (1 alive, 2 died),
 * all zero in every band but the owner's, so the integer sum is an exact merge (and keeps -0.0 and NaN payloads).  The labels
 * of the owned rows are bit-identical to isb_slic_kmeans on the whole image.  Workspace: isb_slic_kmeans_workspace_bytes of
 * the WHOLE image (image_rows, width). */
typedef struct isb_slic_band {
    int32_t slab_rows, width;   /* pixel memory held by this band: rows [y_off, y_off + slab_rows) of the image */
    int32_t image_rows, y_off;
    int32_t own_lo, own_hi;     /* global rows whose clusters this band sums; the bands' [own_lo, own_hi) partition the image */
    int32_t halo;               /* >= 2*step_y; the slab covers [own_lo - halo, own_hi + halo) clipped to the image */
    int32_t n_seeds, step_y, step_x, slic_zero;
    double step;
    const double* lab_slab;     /* plane c, slab row y, column x at lab_slab[c*plane_stride + y*width + x] */
    size_t plane_stride;
    const double* seeds_yx;     /* [n_seeds,2] seeds of the whole image */
    int32_t* labels_slab;       /* [slab_rows, width] */
    void* ws; size_t ws_bytes;
} isb_slic_band_t;
int isb_slic_band_begin(const isb_slic_band_t* band, isb_stream_t stream);
int isb_slic_band_assign(const isb_slic_band_t* band, isb_stream_t stream);
int isb_slic_band_update(const isb_slic_band_t* band, int64_t* xchg, isb_stream_t stream);
int isb_slic_band_import(const isb_slic_band_t* band, const int64_t* xchg, uint64_t* maxdc_xchg /* [n_seeds], SLICO only */,
                         isb_stream_t stream);
int isb_slic_band_finalize(const isb_slic_band_t* band, const uint64_t* maxdc_xchg, isb_stream_t stream);

size_t isb_connectivity_workspace_bytes(int H, int W);


/* _enforce_label_connectivity_cython: raster-order relabel of 4-connected components, BFS truncated at max_size,
 * components < min_size merged into the last already-labelled neighbour seen.  Bit-exact with the oracle.
 *   n_labels_out : device int32, number of output labels (labels are 0..n-1) */
int isb_enforce_connectivity(const int32_t* labels, int H, int W, int min_size, int max_size, int32_t* out,
                             int32_t* n_labels_out, void* ws, size_t ws_bytes, isb_stream_t stream);

/* SLIC of a single-channel VOLUME -- replaces skimage.segmentation.slic(vol, n_segments, compactness, multichannel=False,
 * spacing=space, sigma=1) as called from imsegm/superpixels.py:104-106 (segment_slic_img3d_gray).  Bit-exact with
 * oracle/slic3d_oracle.c.  Written for generality (the reference's volumes are small), see csrc/slic3d.cu.
 *   isb_slic3d_prepare : dtype -> f64 (img_as_float scale for the integer types), scipy gaussian_filter along z, y, x with the
 *                        DEVICE half kernels w_* (radius + 1 weights, [0] = centre; radius 0 / weight 1 = axis not blurred),
 *                        then * ratio (= 1 / compactness).  tmp: scratch of D*H*W doubles
 *   isb_slic3d_kmeans  : the sweeps of _slic_cython; seeds_zyx [n,3] (device); spacing_host: 3 HOST doubles (z, y, x) */
int isb_slic3d_prepare(const void* vol, int dtype, int D, int H, int W, const double* w_z, int r_z, const double* w_y, int r_y,
                       const double* w_x, int r_x, double ratio, double* tmp, double* out, isb_stream_t stream);
size_t isb_slic3d_kmeans_workspace_bytes(int D, int H, int W, int n_seeds);
int isb_slic3d_kmeans(const double* vol_scaled, int D, int H, int W, const double* seeds_zyx, int n_seeds, int step_z, int step_y,
                      int step_x, double step, const double* spacing_host, int max_iter, int32_t* labels, void* ws, size_t ws_bytes,
                      isb_stream_t stream);

/* Slab form of the 3-D sweeps: one volume cut into z-slabs, one (or a few) per GPU, as isb_slic_band_* cuts an image into row
 * bands.  isb_slic3d_prepare_slab blurs slices [z_off, z_off + S) of a volume of depth D (z reflects at the volume's borders, not
 * the slab's); the slices within r_z of either end of an interior slab are not exact, so a caller hands it its k-means slab +-
 * r_z slices (clipped to the volume) and keeps the k-means slab.  The cluster state is replicated in every slab's workspace and
 * lives in the coordinates of the whole volume; a slab assigns every voxel of its k-means slab -- its owned slices + halo, clipped
 * -- from every alive cluster whose +-2*step window meets it, and sums the clusters whose centre slice it owns (all their members
 * are inside the slab; a cluster with a member beyond +-halo slices of its centre -- a voxel that no window reached kept its old
 * label -- is counted in xchg[5 n_seeds] and the caller must then redo the sweeps on the whole volume).  Per sweep:
 *     isb_slic3d_slab_assign -> isb_slic3d_slab_update(xchg) -> [sum xchg as int64 over the slabs] -> isb_slic3d_slab_import(xchg)
 * xchg is [5*n_seeds + 1] int64: per cluster the bit patterns of (cz, cy, cx, cv) and an alive flag (1), all zero in every slab
 * but the owner's and zero for a cluster that died, so the integer sum is an exact merge.  There is no SLICO in 3-D, hence no
 * finalize step.  The labels of the k-means slab are bit-identical to isb_slic3d_kmeans on the whole volume.
 * Workspace: isb_slic3d_kmeans_workspace_bytes(slab_slices, height, width, n_seeds). */
int isb_slic3d_prepare_slab(const void* vol, int dtype, int S, int H, int W, int z_off, int D, const double* w_z, int r_z,
                            const double* w_y, int r_y, const double* w_x, int r_x, double ratio, double* tmp, double* out,
                            isb_stream_t stream);
typedef struct isb_slic3d_slab {
    int32_t depth, height, width;   /* the whole volume */
    int32_t z_off, slab_slices;     /* voxel memory held by this slab: slices [z_off, z_off + slab_slices) (its k-means slab) */
    int32_t own_lo, own_hi;         /* global slices whose clusters this slab sums; the slabs' [own_lo, own_hi) partition the volume */
    int32_t halo;                   /* >= 2*step_z; the slab covers [own_lo - halo, own_hi + halo) clipped to the volume */
    int32_t n_seeds, step_z, step_y, step_x;
    double step;
    double spacing[3];              /* (z, y, x) weights of the spatial distance */
    const double* vol_slab;         /* [slab_slices, height, width] prepared (blurred, * 1/compactness) voxels */
    const double* seeds_zyx;        /* [n_seeds, 3] seeds of the whole volume */
    int32_t* labels_slab;           /* [slab_slices, height, width] */
    void* ws; size_t ws_bytes;
} isb_slic3d_slab_t;
int isb_slic3d_slab_begin(const isb_slic3d_slab_t* slab, isb_stream_t stream);
int isb_slic3d_slab_assign(const isb_slic3d_slab_t* slab, isb_stream_t stream);
int isb_slic3d_slab_update(const isb_slic3d_slab_t* slab, int64_t* xchg, isb_stream_t stream);
int isb_slic3d_slab_import(const isb_slic3d_slab_t* slab, const int64_t* xchg, isb_stream_t stream);

/* _enforce_label_connectivity_cython on a volume (6 neighbours in the order x+1, x-1, y+1, y-1, z+1, z-1).  The workspace
 * grows with D*H*W only; max_size does not change it. */
size_t isb_connectivity3d_workspace_bytes(int D, int H, int W, int max_size);
int isb_enforce_connectivity3d(const int32_t* labels, int D, int H, int W, int min_size, int max_size, int32_t* out,
                               int32_t* n_labels_out, void* ws, size_t ws_bytes, isb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * (ii) descriptors -- replaces imsegm/features_cython.pyx (the reference's only native module)
 * ------------------------------------------------------------------------------------------------------------------ */

/* computeColorImage2dMean :81, ...Energy :101, ...Variance :122 and normColorFeatures :59 in one launch family,
 * plus the centroids of imsegm/superpixels.py:205-224.  Pixels are converted to f32 (descriptors.py:233),
 * accumulated in f64: per-column runs, summed across the lanes of a warp, then the correctly rounded sum of those partials
 * per label, so a rerun on the same input gives the same bits.  At most 2^31 pixels per call.
 *   img     : [H,W,3] interleaved, dtype = isb_dtype (NaN -> 0 as descriptors.py:824)
 *   seg     : [H,W] i32 in [0, nb)
 *   flags   : bit0 mean, bit1 std, bit2 energy  -> feature columns in that order, 3 channels each
 *   feat    : out [nb, ld] f64, columns written at col0.. ; absent labels give 0
 *   centres : optional out [nb,2] f64 (row, col), (-1,-1) for absent labels;  counts: optional out [nb] i32 */
size_t isb_segment_stats_workspace_bytes(int nb);
int isb_segment_stats_2d(const void* img, int dtype, const int32_t* seg, int H, int W, int nb, int flags, double* feat,
                         int ld, int col0, double* centres, int32_t* counts, void* ws, size_t ws_bytes, isb_stream_t stream);

/* The same statistics with caller-owned accumulators, so that row bands of one image can be merged by a collective between
 * the calls: acc [nb,6] f64 (sum c0..c2, sum of squares c0..c2), iacc [nb,3] i64 (count, sum row, sum col), var [nb,3] f64
 * (squared deviations from the f32 mean).  accumulate / deviation ADD into acc+iacc / var (the caller zeroes them), one f64
 * add per entry of the band's rounded sums, so a rerun with the same bands gives the same bits (other bands, other bits);
 * rows are global rows [y_off, y_off + H) of the image for the row sums.  The band's exact sums (484 B per label for accumulate,
 * 244 B for deviation) are allocated and freed on `stream` within the call (cudaMallocAsync / cudaFreeAsync). */
int isb_segment_stats_accumulate(const void* img, int dtype, const int32_t* seg, int H, int W, int y_off, int nb, double* acc,
                                 int64_t* iacc, isb_stream_t stream);
int isb_segment_stats_deviation(const void* img, int dtype, const int32_t* seg, int H, int W, int nb, const double* acc,
                                const int64_t* iacc, float* meanf_scratch /* [nb,3] */, double* var, isb_stream_t stream);
int isb_segment_stats_finish(int nb, int flags, const double* acc, const double* var, const int64_t* iacc, double* feat, int ld,
                             int col0, double* centres, int32_t* counts, isb_stream_t stream);

/* computeGrayImage3dMean :144 / Energy :169 / Variance :194 of features_cython.pyx: one channel, any rank (n <= 2^31 voxels).
 * Runs of 16 voxels, then the correctly rounded sum of their partials per label: a rerun gives the same bits.
 *   flags bit0 mean, bit1 std, bit2 energy -> columns col0.. of feat [nb, ld] in that order */
size_t isb_gray_stats_workspace_bytes(int nb);
int isb_gray_stats(const void* img, int dtype, const int32_t* seg, long long n, int nb, int flags, double* feat, int ld, int col0,
                   void* ws, size_t ws_bytes, isb_stream_t stream);
/* The same statistics with caller-owned accumulators, so that z-slabs of one volume can be merged by a collective between the
 * calls (isb_gray_stats runs exactly these three steps): acc [nb,2] f64 (sum, sum of squares), cnt [nb] i64, var [nb] f64
 * (squared deviations from the f32 mean).  accumulate / deviation ADD into acc+cnt / var (the caller zeroes them), one f64 add
 * per entry of the slab's rounded sums; the slab's exact sums are allocated and freed on `stream` within the call, as above. */
int isb_gray_stats_accumulate(const void* img, int dtype, const int32_t* seg, long long n, int nb, double* acc, int64_t* cnt,
                              isb_stream_t stream);
int isb_gray_stats_deviation(const void* img, int dtype, const int32_t* seg, long long n, int nb, const double* acc, const int64_t* cnt,
                             float* meanf_scratch /* [nb] */, double* var, isb_stream_t stream);
int isb_gray_stats_finish(int nb, int flags, const double* acc, const double* var, const int64_t* cnt, double* feat, int ld, int col0,
                          isb_stream_t stream);

/* computeLabelHistogram2d (features_cython.pyx:222): hist[l] = #{p : segm_select[p] == l >= 0 and struc_elem[p] == 1} */
int isb_label_hist_2d(const int16_t* segm_select, const int16_t* struc_elem, int H, int W, int nb_labels, uint32_t* hist,
                      isb_stream_t stream);

/* histogram_regions_labels_counts (imsegm/labeling.py:208-240, a per-pixel Python loop in the reference): joint histogram
 * hist[a][b] = #{p : slic[p] == a and annot[p] == b}, hist is [nb_slic, nb_annot] u32; labels must be below nb_slic / nb_annot.
 * A pixel with a negative label in either map is skipped, as compute_labels_overlap_matrix (labeling.py:490-523) does. */
int isb_region_label_hist(const int32_t* slic, const int32_t* annot, int H, int W, int nb_slic, int nb_annot, uint32_t* hist,
                          isb_stream_t stream);

/* compute_img_filter_response2d / 3d (imsegm/descriptors.py:951-983): per slice of img [n_slices, H, W] f64 the maximum over a
 * battery of kernels [n_kernels, kh, kw] f64 (odd sizes) of scipy.ndimage.convolve(slice, kernel) -- true convolution, mode
 * 'reflect'.  Generic FP64 utility for the gray-volume texture path; colour images use isb_lm_texture. */
int isb_filter_response_2d(const double* img, int n_slices, int H, int W, const double* kernels, int n_kernels, int kh, int kw,
                           double* out, isb_stream_t stream);

/* scipy.ndimage.gaussian_filter of every slice of img [n_slices, H, W] f64 (rows, then columns; symmetric 1-D correlate, mode
 * 'reflect'), what image_subtract_gauss_smooth (:986-1000) subtracts.  w_half: DEVICE, radius + 1 weights, [0] = centre;
 * tmp: scratch of the image's size */
int isb_gaussian_filter_2d(const double* img, int n_slices, int H, int W, const double* w_half, int radius, double* tmp, double* out,
                           isb_stream_t stream);

/* Inputs of the colour-space groups and of the median / meanGrad statistics of compute_selected_features_color2d, for the
 * resident feature table.  Every launch below is capturable in a CUDA graph (no host read, no allocation). */
enum isb_color_space { ISB_COLOR_HSV = 0, ISB_COLOR_LUV = 1, ISB_COLOR_LAB = 2, ISB_COLOR_HED = 3, ISB_COLOR_XYZ = 4 };
/* convert_img_color_from_rgb (pyimsegm_b200/color.py): img [n_px, 3] interleaved RGB of any isb_dtype (u8 / 255, u16 / 65535,
 * floats as they are) -> out [n_px, 3] f64 in the given isb_color_space.  IEEE pow / cbrt / log; hsv is bit-exact, a NaN pixel
 * gives (0, 0, 0) in hsv. */
int isb_color_convert(const void* img, int dtype, long long n_px, int space, double* out, isb_stream_t stream);
/* np.sum(np.gradient(np.nan_to_num(img[..., c])), axis=0) of every channel of img [H, W, channels] interleaved: one-sided
 * differences at the borders, central halves inside.  out [H, W, channels] is f32 for an f32 image (f32 arithmetic), f64 otherwise
 * (integers are promoted as numpy does).  H < 2 or W < 2 is an argument error, as np.gradient raises. */
int isb_gradient_sum_2d(const void* img, int dtype, int H, int W, int channels, void* out, isb_stream_t stream);
/* isb_segment_median of an [H, W, channels] image into columns col0 .. col0 + channels of the feature table feat [nb, ld]; pixels
 * go through np.nan_to_num first and the result through the table's rules (inf -> largest finite value, -0 -> +0); NaN for a
 * label without pixels.  Workspace: isb_segment_median_workspace_bytes(H * W, nb). */
int isb_segment_median_2d(const void* img, int dtype, const int32_t* seg, int H, int W, int channels, int nb, double* feat, int ld,
                          int col0, void* ws, size_t ws_bytes, isb_stream_t stream);

/* The Leung-Malik route of the statistics the fused kernel does not produce (median, meanGrad): every filter response in memory
 * (texture.py device_lm_materialised).
 * background: planar [3, H, W] f64 = the image [H, W, 3] (any isb_dtype, values as they are) minus its background --
 *   isb_gaussian_filter_2d (w_half DEVICE, radius) of every channel, mixed across the channels by mix [3][3] (HOST, row-major);
 *   tmp and smooth: scratch [3, H, W] f64 */
int isb_lm_background(const void* img, int dtype, int H, int W, const double* w_half, int radius, const double* mix, double* planar,
                      double* tmp, double* smooth, isb_stream_t stream);
/* one battery: resp [3, H, W] = isb_filter_response_2d(planar, kernels [n_kernels, kh, kw]); then clipped at max_signal, its norm
 * |r| = sqrt(sum r^2) summed in a fixed order, and out [H, W, 3] f64 = (r * (log(1 + |r|) / 0.03)) / |r|, or zeros when |r| is 0
 * or infinite */
size_t isb_lm_battery_workspace_bytes(void);
int isb_lm_battery_response(const double* planar, int H, int W, const double* kernels, int n_kernels, int kh, int kw, double max_signal,
                            double* resp, double* out, void* ws, size_t ws_bytes, isb_stream_t stream);
/* The same battery step split in two for row bands of one image (pyimsegm_b200/tiled.py), whose norm is summed over the bands in
 * between.  planar [3, H, W] is a slab of the background-subtracted image.
 * partial: resp [3, H, W] = isb_filter_response_2d(planar, kernels), and *sumsq (DEVICE, one f64) = the sum of the squared responses
 *   clipped at max_signal over the slab rows [row_lo, row_hi) only -- the rows the band owns -- in the fixed block-partial order of
 *   isb_lm_battery_response (a slab that owns all its rows gets that call's sum bit for bit).  Workspace:
 *   isb_lm_battery_workspace_bytes().
 * scale: out [row_hi - row_lo, W, 3] f64 = (r * (log(1 + |r|) / 0.03)) / |r| of the clipped responses resp [3, H, W] of the slab rows
 *   [row_lo, row_hi), with |r| = sqrt(*sumsq) (DEVICE), or zeros when |r| is 0 or infinite */
int isb_lm_battery_partial(const double* planar, int H, int W, const double* kernels, int n_kernels, int kh, int kw, double max_signal,
                           int row_lo, int row_hi, double* resp, double* sumsq, void* ws, size_t ws_bytes, isb_stream_t stream);
int isb_lm_battery_scale(const double* resp, int H, int W, int row_lo, int row_hi, double max_signal, const double* sumsq, double* out,
                         isb_stream_t stream);

/* compute_label_histograms_positions (imsegm/descriptors.py:1288-1352) in one launch: for every position (row, col) and every
 * diameter d the histogram of the labels under the disc dy^2 + dx^2 <= d^2 (skimage.morphology.disk(d)) clipped to the image,
 * i.e. what compute_label_hist_segm (:1396) returns for the pair, and the pixel count of the clipped disc.
 *   segm  : [H, W] i32 labels, values outside [0, nb_labels) ignored;  or proba [H, W, nb_labels] f64 (then segm may be NULL):
 *           hist[l] = sum of proba[.., l] under the disc (compute_label_hist_proba :1501)
 *   positions [n_pos, 2] i32 (row, col), diameters [n_diam] i32;  hist out [n_pos, n_diam, nb_labels] f64, sizes out [n_pos, n_diam] f64
 *   selem : optional explicit structuring element [mh, mw] u8 (1 = inside) used instead of the discs (then n_diam must be 1,
 *           diameters may be NULL); mask pixel (iy, ix) lies on image pixel (row - mh/2 + iy, col - mw/2 + ix) as in
 *           adjust_bounding_box_crop (:1355) */
int isb_disc_label_hist(const int32_t* segm, const double* proba, int H, int W, const int32_t* positions, int n_pos,
                        const int32_t* diameters, int n_diam, const uint8_t* selem, int mh, int mw, int nb_labels, double* hist,
                        double* sizes, isb_stream_t stream);

/* The disc label counts of isb_disc_label_hist for a label map, from run-length rows (center_detection.cu): the map is encoded as
 * the start column and label of every maximal run of each row (one CTA scan per row, in ws), then one CTA per position counts every
 * diameter, each disc row dy as the clipped lengths of the runs under [col - w, col + w], w = floor(sqrt(d^2 - dy^2)) in integers.
 * Same arguments, counts and output layout as isb_disc_label_hist's label-map case (values outside [0, nb_labels) are skipped but
 * count in the size; the disc is clipped to the image; nb_labels <= 4096).  ws: isb_label_runs_workspace_bytes(H, W), 8 H W bytes
 * and some -- sized by the image, not by the label count. */
size_t isb_label_runs_workspace_bytes(int H, int W);
int isb_ring_label_hist(const int32_t* segm, int H, int W, const int32_t* positions, int n_pos, const int32_t* diameters, int n_diam,
                        int nb_labels, double* hist, double* sizes, void* ws, size_t ws_bytes, isb_stream_t stream);

/* sklearn.cluster.DBSCAN(eps, min_samples).fit(points).labels_ for n float64 points [n, 2] (Euclidean): neighbours are the points
 * with dx * dx + dy * dy <= eps * eps (scikit-learn's KD-tree test), the point itself included; core points have at least
 * min_samples neighbours; clusters are numbered by their smallest core index; a non-core point takes the smallest cluster among its
 * core neighbours, else -1.  labels out [n] i32; centres (optional) out [n, 2] f64, rows [0, n_clusters) = the mean of each
 * cluster's points summed in index order (np.mean(points[labels == c], axis=0)); n_clusters: host int.  The call synchronises
 * the stream.  Non-finite points or eps <= 0 return ISB_ERR_ARG; any finite points and eps are clustered (cells of side about eps,
 * coarser when the points span more than 2^29 of them).  n may be 0.  ws: isb_dbscan_workspace_bytes(n), about 80 n bytes. */
size_t isb_dbscan_workspace_bytes(int n);
int isb_dbscan(const double* points, int n, double eps, int min_samples, int32_t* labels, double* centres, int* n_clusters, void* ws,
               size_t ws_bytes, isb_stream_t stream);

/* computeRayFeaturesBinary2d (features_cython.pyx:239) for n_pos positions at once: out [n_pos, n_ang] f32, -1 where the ray
 * leaves the image, 0 where the position lies inside the border label (edge 'up').  sin_a / cos_a: the f32 sines and cosines
 * of the ray angles as the reference forms them (np.deg2rad of the f32 angle, stored to float).  edge: 1 'up', -1 'down'. */
int isb_ray_features_2d(const int8_t* seg_binary, int H, int W, const int32_t* positions, int n_pos, const float* sin_a,
                        const float* cos_a, int n_ang, int edge, float* out, isb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * (iii) graph + energies + alpha-expansion
 * ------------------------------------------------------------------------------------------------------------------ */

/* make_graph_segm_connect_grid2d_conn4 (imsegm/superpixels.py:157-177) for labels already in [0, nb):
 * unique 4-connected label pairs (a < b) sorted by (b, a).
 *   edges : out [cap,2] i32;  n_edges_out : device int32 (if > cap the call reports ISB_ERR_CAPACITY lazily:
 *           the host must check n_edges_out <= cap) */
size_t isb_adjacency_workspace_bytes(int nb, int cap);
int isb_adjacency_edges(const int32_t* seg, int H, int W, int nb, int32_t* edges, int cap, int32_t* n_edges_out, void* ws,
                        size_t ws_bytes, isb_stream_t stream);

/* the same for a label VOLUME [D, H, W]: 6-connectivity (make_graph_segm_connect_grid3d_conn6, superpixels.py:180-202); same
 * workspace as isb_adjacency_edges.  isb_centroids_3d: centre (z, y, x) of every label, (-1,-1,-1) when absent
 * (superpixel_centers on a volume); ws: 4 * nb uint64 */
int isb_adjacency_edges_3d(const int32_t* seg, int D, int H, int W, int nb, int32_t* edges, int cap, int32_t* n_edges_out, void* ws,
                           size_t ws_bytes, isb_stream_t stream);
int isb_centroids_3d(const int32_t* seg, int D, int H, int W, int nb, double* centres, void* ws, size_t ws_bytes, isb_stream_t stream);

/* compute_unary_cost (imsegm/graph_cuts.py:523-540), compute_edge_weights / compute_edge_model / compute_spatial_dist
 * (:574-657, :383-439, :303-336), create_pairwise_matrix_uniform (:442-456), and pyGCO's float->int conversion.
 *   proba [N,K] f64, edges [E,2] i32 (n_edges read from device n_edges_dev when non-null, else E), centres [N,2] or [N,3] f64
 *   metric : 0 = constant 1, 1 = lT (max_k dp^2), 2 = l1, 3 = l2   -> w = exp(-d / (2 std(d)^2));
 *            4 = edge_w already holds the clamped weights (isb_gc_vector_edge_weights): only edge_cost and the integerisation
 *            are applied (spatial must be 0)
 *   spatial: 0 = off; 1 (or 2) = divide by the relative centroid distance over centres (y, x) [N,2] of a label map, 3 = the same
 *            over centres (z, y, x) [N,3] of a label volume (isb_centroids_3d).  The reference does so for edge_type 'model' and
 *            'spatial' exactly, not for 'model_l1' / 'model_l2' (graph_cuts.py:646)
 *   out: unary [N,K] f64, edge_w [E] f64, and the integerised (unary_i [N,K], edge_wi [E], smooth_i [K,K]) i32 */
int isb_gc_energies(const double* proba, int N, const int32_t* n_nodes_dev /* optional device N */, int K, const int32_t* edges, int E,
                    const int32_t* n_edges_dev,
                    const double* centres, int metric, int spatial, double edge_cost, const double* pairwise /* [K,K] device */,
                    double* unary, double* edge_w, int32_t* unary_i, int32_t* edge_wi, int32_t* smooth_i, void* ws,
                    size_t ws_bytes, isb_stream_t stream);
size_t isb_gc_energies_workspace_bytes(int N, int K, int E);

/* the 'color' and 'features' edge weights of compute_edge_weights (imsegm/graph_cuts.py:621-657) over a device edge table:
 *   vec [nb, ld] f64 (first D columns): the per-label vectors, edges [cap, 2] i32 with the count in the optional device n_edges_dev
 *   (an overflowed table, count > cap, reads no edge), centres [nb, 2] (y, x) f64
 *   metric 2: d = L1 distance of the endpoints' vectors ('color'), 3: L2 distance ('features')
 *   edge_w [cap] f64 out: w = exp(-(d / (2 std(d)^2))) with numpy's population std over the real edges (two deterministic passes,
 *   no host read; std 0 gives numpy's NaN / inf), divided by the relative centroid distance of 'spatial', clamped to [1e-3, 1e3]
 *   by comparisons (NaN stays NaN).  isb_gc_energies with metric 4 then integerises edge_w in place.
 *   ws: isb_gc_energies_workspace_bytes(nb, 1, cap) */
int isb_gc_vector_edge_weights(const double* vec, int nb, int D, int ld, const int32_t* edges, int cap, const int32_t* n_edges_dev,
                               const double* centres, int metric, double* edge_w, void* ws, size_t ws_bytes, isb_stream_t stream);
/* np.array(img, dtype=float) of n samples, divided by 255 when minmax[1] (device; isb_image_minmax's maximum) > 1: the image
 * compute_edge_weights takes the 'color' means of.  A NaN maximum compares false and leaves the image unscaled, as np.max does. */
int isb_image_unit_scale(const void* img, int dtype, long long n, const double* minmax, double* out, isb_stream_t stream);

/* gco.cut_general_graph(..., algorithm='expansion', n_iter) on integer energies (imsegm/graph_cuts.py:735-744).
 * One CTA cluster per graph; push-relabel max-flow; a site keeps its label iff it can reach the sink in the
 * residual graph (BK's SINK segment) so labels are identical to the oracle's.
 *   labels : in/out [N] i32 (initial labeling, zeros for the reference call);  energy_out : device int64 */
size_t isb_alpha_expansion_workspace_bytes(int N, int K, int E);
int isb_alpha_expansion(int N, const int32_t* n_nodes_dev /* optional device N */, int K, int E, const int32_t* n_edges_dev,
                        const int32_t* edges, const int32_t* edge_wi,
                        const int32_t* unary_i, const int32_t* smooth_i, int n_iter, int32_t* labels, int64_t* energy_out,
                        int32_t* stats_out /* optional [8]: moves, flows, sweeps, global relabels, BFS levels, smem flag,
                                              a move refused for a terminal capacity >= 2^29, one refused for a pair capacity >= 2^30 */, void* ws, size_t ws_bytes,
                        isb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * class model -- replaces the host round trip of estim_class_model / predict_proba (imsegm/graph_cuts.py:73-163 default
 * 'GMM', imsegm/pipelines.py:95-96) for either mixture of the reference's estim_model variants: StandardScaler +
 * sklearn-style full-covariance EM, n_init restarts run concurrently (one CTA each), best lower bound wins.
 *   kind 0 = GaussianMixture, 1 = BayesianGaussianMixture (full covariance, dirichlet_process, default priors: weight
 *   concentration 1/K, mean precision 1, mean = mean of the scaled features, degrees of freedom D, covariance = their np.cov)
 *   feat [N, ld] f64 (first D columns used), n_dev: optional device int32 with the real row count (<= N)
 *   init_labels: optional [n_init, N] i32 hard assignments (deterministic start); else k-means++/Lloyd from `seed`
 *   proba: out [N, K];  params_out: optional, isb_mixture_fit_params_len(kind, D, K) doubles:
 *     scaler mean[D] | scaler scale[D] | weights[K] | means[K,D] | covariances[K,D,D] | precisions_cholesky[K,D,D] |
 *     lower_bound | n_iter | converged | ok | best_init
 *   For kind 1 the layout has nk (responsibility sums + 10 eps) in place of the weights, the posterior means and (normalised)
 *   covariances, the ELBO as lower_bound, followed by mean_prior[D] | covariance_prior[D,D].
 * ------------------------------------------------------------------------------------------------------------------ */
size_t isb_mixture_fit_workspace_bytes(int kind, int N, int D, int K, int n_init);
int isb_mixture_fit_params_len(int kind, int D, int K);
int isb_mixture_fit_predict(int kind, const double* feat, int N, int D, int ld, const int32_t* n_dev, int K, int n_init, int max_iter,
                            double tol, double reg_covar, int use_scaler, unsigned long long seed, const int32_t* init_labels, double* proba,
                            double* params_out, void* ws, size_t ws_bytes, isb_stream_t stream);
/* PCA fit of the reference's pca_coef (sklearn PCA, covariance_eigh solver) on StandardScaler'd features (use_scaler 0: as given):
 *   n_components > 0 keeps that many components (<= D); else coef in (0, 1) picks them from the explained variance ratio.
 *   params_out (isb_pca_params_len(D) doubles): scaler mean[D] | scaler scale[D] | mean_[D] | components_[D,D] (all of them,
 *   descending, sign-flipped) | explained_variance_[D] | explained_variance_ratio_[D] | singular_values_[D] | mean_ components_^T [D] |
 *   n_components | noise_variance | n_samples | ok;  n_components_out: optional device int32.  The transform is isb_class_transform
 *   with these tables.  D <= 232 (else ISB_ERR_UNSUPPORTED), N >= 2. */
/* sklearn StandardScaler().fit_transform of feat [N, ld] f64 (first D columns; the real row count from the optional device n_dev), bit
 * for bit: the mean and the corrected two-pass variance in numpy's summation order (row after row for D > 1, pairwise for D == 1),
 * _is_constant_feature's scale 1.  The mixture fit's scaler kernel in its exact mode.  params_out [2 D]: mean_ | scale_;
 * out [N, D] = (x - mean_) / scale_ (rows past the real count untouched). */
int isb_standard_scaler(const double* feat, int N, int D, int ld, const int32_t* n_dev, double* params_out, double* out, isb_stream_t stream);
size_t isb_pca_workspace_bytes(int N, int D);
int isb_pca_params_len(int D);
int isb_pca_fit(const double* feat, int N, int D, int ld, const int32_t* n_dev, int use_scaler, double coef, int n_components,
                double* params_out, int32_t* n_components_out, void* ws, size_t ws_bytes, isb_stream_t stream);

/* predict_proba of a caller-fitted class model -- replaces the host round trip of segment_color2d_slic_features_model_graphcut
 * (imsegm/pipelines.py:160-241) with a model from estim_model_classes_group (:113-157) or a trained classifier
 * (imsegm/classification.py:101).  The tables come from pyimsegm_b200/class_models.py; every call is timed under the 'gmm' stage.
 * Rows are [N, ...] with the real row count read from the optional device int32 n_dev (<= N); nothing syncs or allocates.
 *
 * isb_class_transform: the model's feature transform.  out[n] = PCA(scaler(x[n])) with NaN -> 0 first;
 *   feat [N, ld] f64 (first D_in columns); sc_mean / sc_scale: optional [D_in] ((x - mean) / scale, either may be NULL);
 *   pca_comp: optional [D_out, D_in] components_, then pca_mean [D_out] = mean_ components_^T and pca_scale: optional [D_out]
 *   (whitening, sqrt(explained_variance_) clipped at eps); without PCA D_out == D_in.  ws: isb_class_transform_workspace_bytes. */
size_t isb_class_transform_workspace_bytes(int N, int D_in, int has_pca);
int isb_class_transform(const double* feat, int N, int ld, const int32_t* n_dev, int D_in, const double* sc_mean, const double* sc_scale,
                        const double* pca_comp, const double* pca_mean, const double* pca_scale, int D_out, double* out, void* ws,
                        size_t ws_bytes, isb_stream_t stream);
/* Gaussian mixture (GaussianMixture / BayesianGaussianMixture, any covariance type expanded to the full form):
 *   proba[n, k] = softmax_k(log_const[k] - (D log 2 pi + |x[n] U_k - bvec[k]|^2) / 2)
 *   x [N, D] f64; prec_chol [K, D, D] (U_k); bvec [K, D] = means_k U_k; log_const [K] (log-det of U_k + log weight + the BGM terms).
 *   D <= 232, K <= 8 (else ISB_ERR_UNSUPPORTED); D > 16 runs the fit's batched FP64 GEMM in ws (isb_mixture_predict_workspace_bytes). */
size_t isb_mixture_predict_workspace_bytes(int N, int D, int K);
int isb_mixture_predict_proba(const double* x, int N, const int32_t* n_dev, int D, int K, const double* prec_chol, const double* bvec,
                              const double* log_const, double* proba, void* ws, size_t ws_bytes, isb_stream_t stream);
/* decision tree / random forest / extra trees (single output): n_trees trees in structure-of-arrays node tables of n_nodes entries
 * (children as global node indices, -1 at a leaf), tree e starting at roots[e]; value [n_nodes, K] the leaf class fractions.
 * A sample goes left iff (double)(float)x[feature] <= threshold (sklearn's float32 input).  proba = the leaf values added in tree
 * order, divided by n_trees when average != 0: bit-identical to ForestClassifier.predict_proba with n_jobs=None.  K <= 64.
 *   ws: isb_forest_predict_workspace_bytes(N, n_trees) (the leaf of every (sample, tree)) */
size_t isb_forest_predict_workspace_bytes(int N, int n_trees);
int isb_forest_predict_proba(const double* x, int N, const int32_t* n_dev, int D, int n_trees, const int32_t* roots, const int32_t* feature,
                             const double* threshold, const int32_t* left, const int32_t* right, int n_nodes, const double* value, int K,
                             int average, double* proba, void* ws, size_t ws_bytes, isb_stream_t stream);
/* k-nearest neighbours (KNeighborsClassifier, Euclidean metric): fit_x [N_t, D] the training rows (_fit_X), y [N_t] their class
 * indices (_y, in [0, K)).  The squared distance of a query to a training row is sum_d (x_d - t_d)^2 in feature order, every step
 * rounded (no FMA): the bits of a left-to-right float64 loop.  The neighbours are the k smallest by (squared distance, training
 * index).  weights 0 (uniform): proba = class counts / k.  weights 1 (distance): w = 1 / sqrt(d^2), or the indicator d^2 == 0 when
 * any neighbour is at distance 0 (_get_weights); the weights are added per class in ascending neighbour order and divided by their
 * row sum.  1 <= k <= 64, k <= N_t, K <= 64.  ws: isb_knn_predict_workspace_bytes(N, N_t, k) (the per-split neighbour lists). */
size_t isb_knn_predict_workspace_bytes(int N, int N_t, int k);
int isb_knn_predict_proba(const double* x, int N, const int32_t* n_dev, int D, const double* fit_x, int N_t, const int32_t* y, int k, int K,
                          int weights, double* proba, void* ws, size_t ws_bytes, isb_stream_t stream);
/* logistic regression: coef [n_coef, D], intercept [n_coef]; decision_c = x . coef_c + intercept_c.  n_coef == 1 (binary):
 * proba [N, 2] = [1 - expit(d), expit(d)] (_predict_proba_lr); else proba [N, n_coef] = softmax(d) in sklearn.utils.extmath.softmax's
 * order (subtract the row maximum, exp, divide by the row sum).  n_coef <= 64.  ws: isb_linear_predict_workspace_bytes (0 bytes;
 * ws may be NULL). */
size_t isb_linear_predict_workspace_bytes(int N, int n_coef);
int isb_linear_predict_proba(const double* x, int N, const int32_t* n_dev, int D, const double* coef, const double* intercept, int n_coef,
                             double* proba, void* ws, size_t ws_bytes, isb_stream_t stream);

/* compute_texture_desc_lm_img2d_clr (imsegm/descriptors.py:1041-1106): sigma-150 background subtraction (reflect, all three
 * axes), Leung-Malik filter bank (33x33 kernels) as an implicit GEMM on the tensor cores (wgmma.mma_async with TF32 inputs and the 3xTF32
 * split, FP32 accumulators in registers, operands staged by TMA), max over the orientations of a battery, clip at 1e6,
 * log-norm scaling, per-superpixel mean / std / energy -- the responses never leave the SM.
 *   bg_weights : device, 2*bg_radius+1 doubles (scipy's gaussian kernel, sigma 150 -> radius 600); bg_radius 0 = no background
 *   chmix_host : HOST, 3x3 doubles: the same kernel folded onto the reflected length-3 channel axis
 *   w_tc       : device f32 [33 kernel rows][hi | lo][10 k-chunks][NP/8][8 filters][4 taps]: correlation-form (flipped) kernels in
 *                the operand layout of the contraction (K-major 8 x 16-byte core matrices), tf32-rounded value and tf32-rounded
 *                remainder, taps 33..39 and padding filters zero.  Filter (column) order: oriented batteries first (edge s0 |
 *                bar s0 | edge s1 | ..., `orient` filters each), then gauss / LoG / LoG2 per sigma
 *   (orient, NP, n_batt) = (8, 80, 20) full bank | (4, 48, 15) short bank;  flags as isb_segment_stats_2d
 *   feat       : out [nb, ld]: columns col0 + battery*3*nflags + stat*3 + channel (the reference's order) */
size_t isb_lm_workspace_bytes(int H, int W, int nb, int n_batt);
int isb_lm_texture(const void* img, int dtype, const int32_t* seg, int H, int W, int nb, const double* bg_weights, int bg_radius,
                   const double* chmix_host, const float* w_tc, int NP, int orient, int n_batt, int flags,
                   double* feat, int ld, int col0, void* ws, size_t ws_bytes, isb_stream_t stream);
/* The same descriptor for ONE image cut into row bands over several GPUs (SURVEY 8(e), "one huge image"): every band runs
 * isb_lm_texture_accumulate on its slab [slab_rows, W, 3] = the rows it owns, [y_first, y_end) in slab coordinates, plus a halo of
 * bg_radius + 16 rows on every side that is not an image border (at a border the slab ends and reflects like the image); seg points
 * at the slab's first row of the label map.  The sums of the owned rows are ADDED to acc (isb_lm_acc_doubles(nb, n_batt) doubles:
 * sum r | sum r^2 | per-battery global sum r^2) and counts [nb] -- the caller zeroes them, sums them over the bands (all_reduce),
 * and isb_lm_texture_finish forms the same features isb_lm_texture writes. */
size_t isb_lm_acc_doubles(int nb, int n_batt);
int isb_lm_texture_accumulate(const void* img, int dtype, const int32_t* seg, int slab_rows, int W, int y_first, int y_end, int nb,
                              const double* bg_weights, int bg_radius, const double* chmix_host, const float* w_tc, int NP, int orient,
                              int n_batt, double* acc, int32_t* counts, void* ws, size_t ws_bytes, isb_stream_t stream);
int isb_lm_texture_finish(int nb, int n_batt, int flags, const double* acc, const int32_t* counts, double* feat, int ld, int col0,
                          isb_stream_t stream);

/* known-answer test of the tensor-core plumbing (tests/test_gpu_umma.py): D[128, N] = A[128, K] * B[N, K]^T with wgmma.mma_async
 * (TF32 inputs, FP32 accumulators) in one CTA of two warpgroups; A, B row-major f32 holding tf32-representable values,
 * N in {48, 80} (the widths of the contraction), K % 8 == 0 (<= 64).  A comes from registers and B from K-major unswizzled shared
 * memory, the form the contraction uses; variant must be 2 (the shared-memory A operands 0 / 1 are gone). */
int isb_wgmma_selftest(const float* A, const float* B, int N, int K, int variant, float* D, isb_stream_t stream);

/* per-segment, per-channel median -- numpy_img2d_color_median (imsegm/descriptors.py:420-455, channels = 3, n_px = H*W) and
 * numpy_img3d_gray_median (:651-676, channels = 1, n_px = D*H*W); np.median semantics in the image's own type: an odd count gives
 * the middle value, an even count the mean of the two middle values taken in float32 for an ISB_F32 image (sum rounded to float32,
 * then halved) and in float64 otherwise; NaN for a label with a NaN pixel and for a label without pixels.
 *   img : [n_px, channels] interleaved, dtype = isb_dtype;  seg : [n_px] labels in [0, nb);  out : [nb, channels] f64 */
size_t isb_segment_median_workspace_bytes(long long n_px, int nb);
int isb_segment_median(const void* img, int dtype, const int32_t* seg, long long n_px, int channels, int nb, double* out, void* ws,
                       size_t ws_bytes, isb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * (x) ellipse fitting -- imsegm/ellipse_fitting.py: EllipseModelSegm (skimage.measure.EllipseModel + criterion :76-139),
 *     ransac_segm :142-261 and add_overlap_ellipse :282-349
 * ------------------------------------------------------------------------------------------------------------------ */

/* T trials in one launch, one CTA each.  Trial t belongs to centre trial_centre[t] (< C), whose boundary points are
 * pts[pt_off[c] .. pt_off[c+1]) ([P, 2] f64).  Without params_in the trial fits an ellipse (Halir-Flusser direct fit) to the points
 * samp_idx[samp_off[t] .. samp_off[t+1]) (indices into its centre's points, in drawn order); with params_in [T, 5] it takes those
 * parameters.  Then: residuals of every point of the centre (stationary distance from the skimage start angle), n_inl = count of
 * residuals < thr, crit = sum of lab_term[sp_lab[j]] over the N superpixel points sp_pts [N, 2] inside the ellipse, added in a fixed
 * order.  ok [T]: 1 fitted, 0 not exactly one admissible eigenvector, -1 singular S3 (numpy's LinAlgError).  params_out [T, 5];
 * resid_out (optional): residuals of trial t at resid_out[resid_off[t] ..].  The caller validates sample indices. */
int isb_ellipse_ransac(int T, const int32_t* trial_centre, const int32_t* samp_off, const int32_t* samp_idx, const double* params_in,
                       int C, const double* pts, const int32_t* pt_off, double thr, const double* sp_pts, const int32_t* sp_lab,
                       const double* lab_term, int N, int32_t* ok, double* params_out, int32_t* n_inl, double* crit,
                       double* resid_out, const long long* resid_off, isb_stream_t stream);
/* skimage.draw.ellipse raster of one ellipse into mask [H, W] u8 and, in the same pass over segm [H, W] i32, counts [2 * n_labels + 1]
 * u64: pixels per label | pixels per label inside the ellipse | ellipse area.  bbox_host (HOST, 4 ints): clipped bounding box
 * r0, c0, r1, c1 (inclusive); geom_host (HOST, 6 doubles): centre relative to (r0, c0), the two radii, sin and cos of the rotation.
 * Labels outside [0, n_labels) are not counted; up to 4096 labels are counted in shared memory, more directly in counts. */
int isb_ellipse_overlap(const int32_t* segm, int H, int W, int n_labels, const int32_t* bbox_host, const double* geom_host,
                        uint8_t* mask, unsigned long long* counts, isb_stream_t stream);
/* grey erosion (op 0) or dilation (op 1) of a 0/1 mask [H, W] u8 over n_offsets (dy, dx) footprint offsets (device i32 [n, 2]),
 * borders as scipy.ndimage's 'reflect'.  Two calls with the offsets of skimage.morphology.disk(r) make the opening that
 * imsegm/descriptors.py:1873-1876 and imsegm/ellipse_fitting.py apply to a binary mask. */
int isb_binary_morph_footprint(const uint8_t* in, int H, int W, const int32_t* offsets, int n_offsets, int op, uint8_t* out,
                               isb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * (x') supervised training data -- the per-image step of train_classif_color2d_slic_features (imsegm/pipelines.py:293-379)
 * ------------------------------------------------------------------------------------------------------------------ */

/* one training label per superpixel: wrapper_compute_color2d_slic_features_labels (pipelines.py:272-290) over
 * histogram_regions_labels_norm (labeling.py:245-278), without the dense [nb, max label + 1] table of isb_region_label_hist.
 *   slic [H, W] i32 in [0, nb) (other values are not counted), annot [H, W] i32 (negative = unknown), labels out [nb] i64.
 * With c* the largest pixel count of a known label in the superpixel, l* the smallest label with that count, u its unknown pixels and
 * n all its pixels: labels[s] = l* when c* >= u and !((double)c* / (double)n < label_purity), else -1 -- the reference's np.argmax,
 * which ranks its unknown bin max(annot) + 1 after every label, and its purity test.  A superpixel without pixels, or at or beyond the
 * optional device count n_labels_dev, gets -1.  Memory and time follow H * W and nb, never the label values: (superpixel, label)
 * pairs are counted in a hash table of 1.5 H W entries.  H * W <= 2^31.  ws: isb_train_labels_workspace_bytes(H, W, nb), 18 bytes
 * per pixel and 16 per superpixel. */
size_t isb_train_labels_workspace_bytes(int H, int W, int nb);
int isb_superpixel_train_labels(const int32_t* slic, int H, int W, int nb, const int32_t* n_labels_dev, const int32_t* annot,
                                double label_purity, int64_t* labels, void* ws, size_t ws_bytes, isb_stream_t stream);

/* balance_dataset_by_(features[labels != -1], labels[labels != -1], 'unique') of one image (classification.py:1159-1216): the rows of
 * feat [N, ld] f64 (first D columns; the real row count from the optional device n_dev) whose label [N] i64 is not -1, each value
 * rounded as rint(x * 1000.0) / 1000.0 (np.round(x, 3), bit for bit), grouped by label ascending, sorted lexicographically within a
 * label and without repeats (-0 equals +0 and is written as +0).  Out: rows_out [N, D] f64 (the first *n_out rows), labels_out [N]
 * i64 (the label of each written row) and n_out (DEVICE i64).  The table must hold no NaN (the pipelines replace NaN by 0 first): a
 * NaN in a kept row sets *n_out to -1, and nothing the call wrote is meaningful.  Nothing synchronises with the host.
 * ws: isb_unique_rows_workspace_bytes(N, D), a rounded copy of the table and some 30 bytes per row. */
size_t isb_unique_rows_workspace_bytes(int N, int D);
int isb_unique_rows_rounded(const double* feat, int N, int D, int ld, const int32_t* n_dev, const int64_t* labels, double* rows_out,
                            int64_t* labels_out, long long* n_out, void* ws, size_t ws_bytes, isb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * (xi) labeling -- imsegm/labeling.py: boundary and contour maps, the exact Euclidean distance transform, the (row, col)
 *      lists of contour_coords / compute_boundary_distances, and the final relabel gather.  Label maps are [H, W] i32.
 * ------------------------------------------------------------------------------------------------------------------ */

/* skimage.segmentation.find_boundaries(seg, mode='thick', connectivity=1) of compute_boundary_distances (labeling.py:708,710):
 * out [H, W] u8 is 1 where one of the pixel's in-image 4-neighbours has another label (pixels outside the image never count,
 * negative labels are ordinary values). */
int isb_label_boundary_map(const int32_t* seg, int H, int W, uint8_t* out, isb_stream_t stream);
/* contour_binary_map (labeling.py:34-79) as 0 / 1 u8: rows 1..H-2 and columns 1..W-2 are 1 where seg == label and a 4-neighbour
 * differs from label; include_boundary != 0 also sets every frame pixel with seg == label. */
int isb_label_contour_map(const int32_t* seg, int H, int W, int32_t label, int include_boundary, uint8_t* out, isb_stream_t stream);
/* scipy.ndimage.distance_transform_edt of an input whose zeros are the nonzero pixels of sites [H, W] u8 (compute_distance_map
 * labeling.py:167, compute_boundary_distances :711): dist [H, W] f64 = sqrt((double)d2), d2 the integer squared distance to the
 * nearest site -- bit-identical to scipy.  Without any site every pixel is measured from (-1, 0), as scipy's feature transform
 * does: dist = sqrt((y + 1)^2 + x^2).  H, W <= 32768 (d2 fits int32), else ISB_ERR_ARG.  ws: isb_edt_workspace_bytes(H, W). */
size_t isb_edt_workspace_bytes(int H, int W);
int isb_edt_2d(const uint8_t* sites, int H, int W, double* dist, void* ws, size_t ws_bytes, isb_stream_t stream);
/* the same transform giving, instead of the distance, the flat index (row * W + column) of a nearest site (image_inpaint_pixels,
 * annotation.py:279-286): index [H, W] i32, -1 everywhere when there is no site.  Of equidistant sites it takes the one of smallest
 * column, then of smallest row -- the choice of scipy.ndimage.distance_transform_edt(..., return_indices=True).  Same kernels as
 * isb_edt_2d plus one byte per pixel; ws: isb_edt_index_workspace_bytes(H, W). */
size_t isb_edt_index_workspace_bytes(int H, int W);
int isb_edt_2d_indices(const uint8_t* sites, int H, int W, int32_t* index, void* ws, size_t ws_bytes, isb_stream_t stream);
/* order-preserving compaction of a mask [H, W] u8 (contour_coords labeling.py:101-105, the point list of
 * compute_boundary_distances :707-712): isb_mask_compact_count scans the per-tile counts into ws and writes the number P of set
 * pixels to the DEVICE int64 total; isb_mask_compact_write (same ws, after the count) writes points [P, 2] i64 (row, col) in raster
 * order and, when values [H, W] f64 is given, values_out [P] = values at those pixels.  ws: isb_mask_compact_workspace_bytes. */
size_t isb_mask_compact_workspace_bytes(int H, int W);
int isb_mask_compact_count(const uint8_t* mask, int H, int W, void* ws, size_t ws_bytes, long long* total, isb_stream_t stream);
int isb_mask_compact_write(const uint8_t* mask, int H, int W, const double* values, const void* ws, size_t ws_bytes, int64_t* points,
                           double* values_out, isb_stream_t stream);
/* the final step of relabel_max_overlap_unique (labeling.py:611-613), relabel_max_overlap_merge (:678-680) and
 * assume_bg_on_boundary (:753): out = lut[seg] where 0 <= seg < n_lut, out = seg elsewhere (negative labels pass through).
 * isb_gather below indexes its table unguarded. */
int isb_relabel_gather(const int32_t* seg, long long npx, const int32_t* lut, int n_lut, int32_t* out, isb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * (xii) annotation -- imsegm/annotation.py: colour histograms, palette lookups and nearest-pixel quantisation.  Pixels are
 *       interleaved [n_px, channels]; label maps are i64.
 * ------------------------------------------------------------------------------------------------------------------ */

/* colour histogram of unique_image_colors / image_frequent_colors (annotation.py:46-68, :163-193): hist [2^24] u64 gets +1 at
 * r << 16 | g << 8 | b for every pixel of img [n_px, channels] u8; channels 3 or 4 (only the first three count), 1 = grey (v, v, v).
 * accumulate = 0 zeroes hist first, 1 adds to what it holds (several images into one histogram). */
int isb_color_hist(const uint8_t* img, long long n_px, int channels, int accumulate, unsigned long long* hist, isb_stream_t stream);
/* the nonzero bins of hist in ascending packed order, as isb_mask_compact_count / _write: the count writes their number P to the
 * DEVICE int64 total, the write (same ws, after the count) colors [P] i32 (packed RGB) and counts [P] i64.
 * ws: isb_color_hist_workspace_bytes(). */
size_t isb_color_hist_workspace_bytes(void);
int isb_color_hist_compact_count(const unsigned long long* hist, void* ws, size_t ws_bytes, long long* total, isb_stream_t stream);
int isb_color_hist_compact_write(const unsigned long long* hist, const void* ws, size_t ws_bytes, int32_t* colors, int64_t* counts,
                                 isb_stream_t stream);
/* palette index of every pixel of img [n_px, channels] (channels 1 .. 4) against palette [n_colors, channels] of the same dtype
 * (ISB_U8 or ISB_F64; n_colors <= 1024, else ISB_ERR_UNSUPPORTED):
 *   mode 0, exact (convert_img_colors_to_labels_reverted :94-125, quantize_image_nearest_pixel :308-316): the LAST entry equal to the
 *           pixel in every channel, -1 when none; unmatched (optional DEVICE u64) gets the number of -1 pixels, matched (optional
 *           [n_px] u8) 1 / 0 per pixel;
 *   mode 1, L1-nearest (image_color_2_labels :245-247, quantize_image_nearest_color :271-273): the FIRST entry of least sum of
 *           |pixel - entry| over the channels (np.argmin); uint8 sums are exact integers, float64 sums add the channels in order from
 *           0 as numpy does, and a NaN distance wins at its first occurrence.
 * labels [n_px] i64 = values[index] when values [n_colors] i64 is given, the index otherwise. */
int isb_palette_map(const void* img, int dtype, long long n_px, int channels, const void* palette, int n_colors, int mode,
                    const int64_t* values, int64_t* labels, uint8_t* matched, unsigned long long* unmatched, isb_stream_t stream);
/* label -> colour gather (convert_img_labels_to_colors :128-160): out [n_px] rows of row_bytes (1 .. 32) bytes = the row of table
 * [n_colors, row_bytes] for each label -- with keys [n_colors] i64 (ascending, unique) the row whose key equals the label, without
 * them row = label for 0 <= label < n_colors.  A label without a row writes zeros and is counted in missing (optional DEVICE u64).
 * n_colors <= 1024, else ISB_ERR_UNSUPPORTED. */
int isb_palette_gather(const int64_t* labels, long long n_px, const int64_t* keys, int n_colors, const void* table, int row_bytes,
                       void* out, unsigned long long* missing, isb_stream_t stream);
/* out[i] = src[index[i]] for n elements of elem_bytes (1, 2, 4 or 8) bytes: the values at the sites of isb_edt_2d_indices
 * (image_inpaint_pixels :279-286).  Indices are not checked. */
int isb_gather_at_index(const void* src, int elem_bytes, const int32_t* index, long long n, void* out, isb_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------------
 * (xiii) classification -- the scoring half of imsegm/classification.py: every metric derives from one contingency table.
 * ------------------------------------------------------------------------------------------------------------------ */

/* contingency table of two label maps y_true, y_pred [n] of dtypes ISB_BOOL, ISB_U8, ISB_I8, ISB_U16, ISB_I16, ISB_I32, ISB_U32 or
 * ISB_I64 (the two may differ): the pixels of every (true value, pred value) pair, leaving out every pixel whose value in either map
 * is one of drop [n_drop] i64 (ascending; optional when n_drop = 0) -- compute_classif_stat_segm_annot :404-410.
 * The count (synchronises the stream twice, to read 4 and 2 values back) writes to the HOST info [6]:
 *   K_true, K_pred (distinct kept values of each map; 0, 0 when every pixel is dropped), min_true, range_true, min_pred, range_pred.
 * The kept values of a map of 32 or 64 bits must span fewer than 2^26 values, else ISB_ERR_UNSUPPORTED.
 * The write (same arguments, info and ws, after the count) writes values_true [K_true] and values_pred [K_pred] i64 ascending and
 * counts [K_true * K_pred] i64, row-major over (true, pred); K_true * K_pred <= 2^28, else ISB_ERR_UNSUPPORTED.
 * ws: isb_contingency_workspace_bytes(dtype_true, dtype_pred) (0 for an unsupported dtype). */
size_t isb_contingency_workspace_bytes(int dtype_true, int dtype_pred);
int isb_contingency_count(const void* y_true, int dtype_true, const void* y_pred, int dtype_pred, long long n, const int64_t* drop, int n_drop,
                          void* ws, size_t ws_bytes, long long* info, isb_stream_t stream);
int isb_contingency_write(const void* y_true, int dtype_true, const void* y_pred, int dtype_pred, long long n, const int64_t* drop, int n_drop,
                          const long long* info, void* ws, size_t ws_bytes, int64_t* values_true, int64_t* values_pred, int64_t* counts,
                          isb_stream_t stream);

/* k-means down-sampling of down_sample_dict_features_kmean (:1110-1134): the Lloyd runs of scikit-learn's
 * KMeans(init='random', n_init=3, max_iter=5) and the sample nearest to each final centre.  X [n, D] f64 row-major, 1 <= k <= n;
 * D <= 256, n <= 2^30 and k <= 4 194 240, else ISB_ERR_UNSUPPORTED.  ws: isb_kmeans_workspace_bytes(n, k, D) (0 out of range).
 *
 * isb_kmeans_lloyd continues one run of _kmeans_single_lloyd (unit weights) on the centred X from centres [k, D] (in / out),
 * labels [n] i32 (in / out; -1 everywhere for a new run) and status [4] i32 (device, in / out; zeros for a new run):
 *   status[0] 0 running, 1 strict convergence, 2 centre shift within tol, 3 stopped on an empty cluster, 4 max_iter sweeps done;
 *   status[1] sweeps done; status[2] labels changed in the current sweep; status[3] empty clusters in the current sweep.
 * A sweep labels every row by argmin_j |c_j|^2 - 2 x.c_j (FP64 tensor cores; lowest j on ties), writes the member sums [k, D] f64
 * (members added in ascending row order) and counts [k] i32, and without an empty cluster sets c_j = sum_j * (1 / count_j), then
 * stops strictly when no label changed or when the sum of squared centre shifts is <= tol.  A run that stops without strict
 * convergence relabels the rows once more; every stopped run writes inertia [1] f64 = sum of (x - c_label)^2.  All of it is enqueued
 * without a host read: the call enqueues `sweeps` sweeps (0 <= sweeps <= max_iter; max_iter - status[1] to finish the run, 0 to only
 * relabel and sum the inertia of a run that has stopped), each of which does nothing once the run has stopped except its radix sort
 * of the n (label, row) pairs.  A sweep with an empty cluster stops with status 3 and leaves labels, sums, counts and the centres it
 * started from; the caller updates the centres, sets status (0 with status[1] + 1 sweeps to go on, or the code it stops with) and
 * calls again.  Every call copies X into the workspace once (rows padded for the tensor-core tiles).  The member sums take one warp
 * per cluster, so their time follows the largest cluster: with k = 1 one warp adds all n rows. */
size_t isb_kmeans_workspace_bytes(int n, int k, int D);
int isb_kmeans_lloyd(const double* X, int n, int D, int k, int max_iter, int sweeps, double tol, double* centres, int32_t* labels, int32_t* status,
                     double* sums, int32_t* counts, double* inertia, void* ws, size_t ws_bytes, isb_stream_t stream);
/* nearest [k] i32: for every centre [k, D] the row of X of least squared distance sum_d (x_d - c_d)^2 (features added in order), the
 * lowest row index among equal distances -- np.argmin(euclidean_distances(X, centres), axis=0) without the expansion's rounding */
int isb_kmeans_nearest(const double* X, int n, int D, const double* centres, int k, int32_t* nearest, void* ws, size_t ws_bytes,
                       isb_stream_t stream);

/* exact-split Gini trees of scikit-learn's DecisionTreeClassifier / RandomForestClassifier fit (splitter 'best'), the classifier
 * that create_classif_search_train_export (:656-759) trains; all T trees of a forest are built together, level by level.
 *   x [n, D] f32 row-major (scikit-learn's trees cast X to float32), y [n] i32 class indices in [0, K), K <= 64;
 *   counts [T, n] i32: the sample weight of every row in every tree (bootstrap counts, or ones); a row of count 0 is not in the tree;
 *   seeds [T] u64 (device): the key of each tree's feature sampling.
 *   max_features m in [1, D], min_samples_split >= 2, min_samples_leaf >= 1 (rows with a nonzero count), max_depth (-1: none),
 *   min_impurity_decrease: the parameters as scikit-learn's fit resolves them.
 * The split rules are scikit-learn 1.9's: Gini proxy improvement from the weighted class counts, positions where the next sorted value is
 * above the previous + 1e-7f (float32) only, both sides >= min_samples_leaf rows, threshold x[p-1] / 2.0 + x[p] / 2.0 in f64, and the
 * leaf tests of the depth-first builder.  Feature sampling differs from scikit-learn's sequential RNG: a node's candidates are the m
 * non-constant features of least (h, feature), h = splitmix64(splitmix64(splitmix64(seed) ^ b) ^ feature) with b the node's
 * breadth-first index in its tree (children of earlier parents first, left before right); equal proxies go to the lowest feature, then
 * the lowest position.
 * Outputs per tree t at [t * cap + node], nodes numbered in preorder (the depth-first builder's ids): left, right, feature (i32; -1, -1,
 * -2 at a leaf), threshold (f64; -2.0 at a leaf), impurity (f64), n_node_samples (i32 rows), weighted_n_node_samples (f64),
 * missing_go_to_left (u8: n_left > n_right at a split, 0 at a leaf), class_counts [.., K] i32 (weighted), node_count [T] i32 (device).
 * cap >= 2 * nnz(counts[t]) - 1 for every t, else ISB_ERR_CAPACITY.  n_levels (host, optional): the levels built.
 * Limits (ISB_ERR_UNSUPPORTED): D <= 2048, T * n * m < 2^31, a row count < 2^24, the total count of a tree < 2^26.
 * The call synchronises the stream: it reads back a few integers per level to size the next launches.
 * ws: isb_forest_fit_workspace_bytes(n, D, T, K, max_features) (0 out of range). */
size_t isb_forest_fit_workspace_bytes(int n, int D, int T, int K, int max_features);
int isb_forest_fit(const float* x, int n, int D, const int32_t* y, int K, const int32_t* counts, int T, const uint64_t* seeds, int max_features,
                   int min_samples_split, int min_samples_leaf, int max_depth, double min_impurity_decrease, int cap, int32_t* left, int32_t* right,
                   int32_t* feature, double* threshold, double* impurity, int32_t* n_node_samples, double* weighted_n_node_samples,
                   uint8_t* missing_go_to_left, int32_t* class_counts, int32_t* node_count, int* n_levels /* host */, void* ws, size_t ws_bytes,
                   isb_stream_t stream);

/* isb_forest_fit for trees of G groups in one call, level by level together: a group is one training set with its own transformed copy of
 * the rows and its own resolved parameters (a cross-validation fold: its scaler / PCA, its max_features and leaf sizes).
 *   x [G, n, Dmax] f32 (device): group g's rows, its features in columns [0, D[g]); columns at or beyond D[g] are never read;
 *   D, max_features, min_samples_split, min_samples_leaf [G] i32 (host): per group, D[g] in [1, Dmax], max_features[g] in [1, D[g]],
 *   min_samples_split[g] >= 2, min_samples_leaf[g] >= 1;
 *   y [n] i32 class indices in [0, K) and K shared by every group (a class missing from a group's rows changes no Gini value);
 *   counts [T, n] i32 (device), seeds [T] u64 (device) and tree_group [T] i32 (host, in [0, G)) per tree: a row outside the tree's
 *   training set has count 0;
 *   max_depth and min_impurity_decrease shared.
 * Every tree is node for node the tree isb_forest_fit builds from its group's x [n, D[g]] and parameters alone.  Outputs, cap and n_levels
 * (the levels of the deepest tree) as isb_forest_fit.  Argument errors (a group or tree index out of range, a parameter outside its range,
 * D[g] > Dmax) return ISB_ERR_ARG before any device work.  Limits (ISB_ERR_UNSUPPORTED): those of isb_forest_fit with D = Dmax and
 * m = max(max_features).
 * ws: isb_forest_fit_groups_workspace_bytes(n, Dmax, G, T, K, max(max_features)) (0 out of range). */
size_t isb_forest_fit_groups_workspace_bytes(int n, int Dmax, int G, int T, int K, int max_features_max);
int isb_forest_fit_groups(const float* x, int n, int Dmax, int G, const int32_t* D /* host */, const int32_t* max_features /* host */,
                          const int32_t* min_samples_split /* host */, const int32_t* min_samples_leaf /* host */, const int32_t* y, int K,
                          const int32_t* counts, int T, const int32_t* tree_group /* host */, const uint64_t* seeds, int max_depth,
                          double min_impurity_decrease, int cap, int32_t* left, int32_t* right, int32_t* feature, double* threshold,
                          double* impurity, int32_t* n_node_samples, double* weighted_n_node_samples, uint8_t* missing_go_to_left,
                          int32_t* class_counts, int32_t* node_count, int* n_levels /* host */, void* ws, size_t ws_bytes, isb_stream_t stream);

/* random-split Gini trees of scikit-learn's ExtraTreesClassifier fit, node for node the trees scikit-learn 1.9 builds (the forest of
 * feature_scoring_selection); one CTA per tree replays the depth-first builder and every draw of its splitter.
 *   x [n, D] f32 row-major, y [n] i32 class indices in [0, K), K <= 64, counts [T, n] i32: as isb_forest_fit;
 *   rand_r_state [T] u32 (device): each tree's splitter state, RandomState(tree seed).randint(0, 2^31 - 1) (Splitter.init);
 *   max_features, min_samples_split, min_samples_leaf, max_depth (-1: none), min_impurity_decrease: as isb_forest_fit;
 *   small_rows: nodes of at most this many rows build their subtree on one warp from rows staged in shared memory (0: the default,
 *   64; lowered until the staged rows fit 96 KiB).
 * The rules are node_split_random's (_splitter.pyx) and DepthFirstTreeBuilder.build's (_tree.pyx): the Fisher-Yates feature draws
 * rand_int(n_drawn_constants, f_i - n_found_constants) with the known / found / drawn constant bookkeeping, the features and
 * constant_features arrays carried from node to node in depth-first order; a feature is constant when max <= min + 1e-7f (float32);
 * threshold rand_uniform(min, max) in f64, min when it equals max; rows with (f64) x <= threshold go left; a candidate with fewer than
 * min_samples_leaf rows on a side is rejected; the largest Gini proxy wins (the first on ties); missing_go_to_left = n_left > n_right;
 * the builder's leaf tests; the left child is built first.  our_rand_r maps a state of 0 to 1.
 * Outputs, their layout and cap: as isb_forest_fit.  Argument errors (including a negative count, a class outside [0, K) or a tree with
 * no row) return ISB_ERR_ARG.  Limits (ISB_ERR_UNSUPPORTED): D <= 2048, K <= 64, T * n < 2^31, the total count of a tree < 2^26.
 * The call synchronises the stream once, before the build, to check the counts.
 * ws: isb_extra_trees_fit_workspace_bytes(n, D, T, K, max_features) (0 out of range), about 28 * T * n bytes. */
size_t isb_extra_trees_fit_workspace_bytes(int n, int D, int T, int K, int max_features);
int isb_extra_trees_fit(const float* x, int n, int D, const int32_t* y, int K, const int32_t* counts, int T, const uint32_t* rand_r_state,
                        int max_features, int min_samples_split, int min_samples_leaf, int max_depth, double min_impurity_decrease,
                        int small_rows, int cap, int32_t* left, int32_t* right, int32_t* feature, double* threshold, double* impurity,
                        int32_t* n_node_samples, double* weighted_n_node_samples, uint8_t* missing_go_to_left, int32_t* class_counts,
                        int32_t* node_count, void* ws, size_t ws_bytes, isb_stream_t stream);

/* dst[0..n) = value (initial labeling of isb_alpha_expansion and similar small fills) */
int isb_fill_i32(int32_t* dst, long long n, int32_t value, isb_stream_t stream);

/* dst[i] = dst[i] (op) src[i] over n 8-byte words; op 0 int64 sum, 1 int64 max, 2 f64 min, 3 f64 max (both NaN when either
 * side is NaN), 4 f64 sum.  What a
 * collective does between GPUs in row-band mode, for several bands held by one GPU. */
int isb_combine(void* dst, const void* src, long long n, int op, isb_stream_t stream);

/* final LUT gathers of imsegm/pipelines.py:104,109:  segm = graph_labels[slic], segm_soft = proba[slic]
 *   lut_i [nb] i32 (optional), lut_p [nb,K] f64 (optional); outputs [H,W] i32 / [H,W,K] f64 */
int isb_gather(const int32_t* seg, long long npx, const int32_t* lut_i, const double* lut_p, int K, int32_t* out_i,
               double* out_p, isb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* IMSEGM_B200_H */
