// ellipse_fit.cu -- RANSAC ellipse fitting of imsegm/ellipse_fitting.py (EllipseModelSegm, ransac_segm) and the ellipse raster of
// add_overlap_ellipse.  One CTA evaluates one trial: the direct fit of its samples, the distance of every boundary point of its
// centre to the ellipse, and the segmentation criterion over every superpixel centre.  All sums run in a fixed order, so a trial
// gives the same bits as the single-model calls (estimate / residuals / criterion) that run through the same kernel as a batch of one.
#include "common.cuh"

namespace {

constexpr int ETHREADS = 128;
constexpr int ELL_SMEM_LABELS = 4096;

struct Fit {
    int status;      // 1 fitted, 0 not exactly one admissible eigenvector, -1 singular S3
    double p[5];     // xc, yc, a, b, theta
};

// inverse of a 3x3 matrix by LU with partial pivoting; false on an exactly zero pivot (numpy.linalg.inv raises there)
__host__ __device__ bool inv3(const double A[3][3], double X[3][3])
{
    double L[3][3];
    int perm[3] = {0, 1, 2};
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) L[i][j] = A[i][j];
    for (int k = 0; k < 3; ++k) {
        int piv = k;
        for (int i = k + 1; i < 3; ++i)
            if (fabs(L[i][k]) > fabs(L[piv][k])) piv = i;
        if (L[piv][k] == 0.0) return false;
        if (piv != k) {
            for (int j = 0; j < 3; ++j) { double t = L[k][j]; L[k][j] = L[piv][j]; L[piv][j] = t; }
            int t = perm[k]; perm[k] = perm[piv]; perm[piv] = t;
        }
        for (int i = k + 1; i < 3; ++i) {
            L[i][k] = L[i][k] / L[k][k];
            for (int j = k + 1; j < 3; ++j) L[i][j] = L[i][j] - L[i][k] * L[k][j];
        }
    }
    for (int c = 0; c < 3; ++c) {
        double y[3];
        for (int i = 0; i < 3; ++i) {
            double s = perm[i] == c ? 1.0 : 0.0;
            for (int j = 0; j < i; ++j) s = s - L[i][j] * y[j];
            y[i] = s;
        }
        for (int i = 2; i >= 0; --i) {
            double s = y[i];
            for (int j = i + 1; j < 3; ++j) s = s - L[i][j] * X[j][c];
            X[i][c] = s / L[i][i];
        }
    }
    return true;
}

__host__ __device__ double nan_to_num(double v)
{
    if (isnan(v)) return 0.0;
    if (isinf(v)) return v > 0 ? 1.7976931348623157e308 : -1.7976931348623157e308;
    return v;
}

// ellipse parameters of the conic coefficients a1 = (a, b, c) and a2 = P a1 (skimage 0.14-0.18 EllipseModel.estimate, as recalled)
__host__ __device__ void conic_params(const double v[3], const double P[3][3], double out[5])
{
    double a = v[0], b = v[1], c = v[2];
    double d = P[0][0] * v[0] + P[0][1] * v[1] + P[0][2] * v[2];
    double f = P[1][0] * v[0] + P[1][1] * v[1] + P[1][2] * v[2];
    double g = P[2][0] * v[0] + P[2][1] * v[1] + P[2][2] * v[2];
    b = b / 2.0; d = d / 2.0; f = f / 2.0;
    const double den = b * b - a * c;
    const double x0 = (c * d - b * f) / den;
    const double y0 = (a * f - b * d) / den;
    const double num = a * (f * f) + c * (d * d) + g * (b * b) - 2.0 * b * d * f - a * c * g;
    const double term = sqrt((a - c) * (a - c) + 4.0 * (b * b));
    const double den1 = den * (term - (a + c));
    const double den2 = den * (-term - (a + c));
    const double width = sqrt(2.0 * num / den1);
    const double height = sqrt(2.0 * num / den2);
    double phi = 0.5 * atan((2.0 * b) / (a - c));
    // a == c puts atan's axis at +-pi/4 on the larger eigenvalue of [[a, b], [b, c]], as a > c does, while width comes from the
    // smaller one for either sign of the eigenvector: turn it by pi / 2 there too (skimage's a > c leaves theta on the other axis)
    if (a >= c) phi += 0.5 * 3.141592653589793;
    out[0] = nan_to_num(x0); out[1] = nan_to_num(y0); out[2] = nan_to_num(width); out[3] = nan_to_num(height); out[4] = nan_to_num(phi);
}

// real eigenvalues of a 3x3 matrix (roots of its characteristic polynomial, Newton-polished); returns how many
__host__ __device__ int eig3_real(const double M[3][3], double lam[3])
{
    const double tr = M[0][0] + M[1][1] + M[2][2];
    const double c1 = M[0][0] * M[1][1] - M[0][1] * M[1][0] + M[0][0] * M[2][2] - M[0][2] * M[2][0] + M[1][1] * M[2][2] - M[1][2] * M[2][1];
    const double det = M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0])
                     + M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
    // lambda^3 - tr lambda^2 + c1 lambda - det; lambda = x + tr / 3
    const double s = tr / 3.0;
    const double p = c1 - tr * tr / 3.0;
    const double q = -2.0 * s * s * s + c1 * s - det;      // x^3 + p x + q = 0
    int n = 0;
    const double disc = (q / 2.0) * (q / 2.0) + (p / 3.0) * (p / 3.0) * (p / 3.0);
    // the pencil of the direct fit has three real eigenvalues: a discriminant that rounding pushed just above zero is a double root
    const double p3 = (p / 3.0) * (p / 3.0) * (p / 3.0);
    if (p < 0 && disc <= -p3 * 1e-12) {
        const double r = 2.0 * sqrt(-p / 3.0);
        double arg = 3.0 * q / (p * r);
        arg = fmin(1.0, fmax(-1.0, arg));
        const double th = acos(arg) / 3.0;
        for (int k = 0; k < 3; ++k) lam[n++] = s + r * cos(th - 2.0 * 3.141592653589793 * k / 3.0);
    } else {
        const double sq = sqrt(fmax(disc, 0.0));
        lam[n++] = s + cbrt(-q / 2.0 + sq) + cbrt(-q / 2.0 - sq);
    }
    for (int k = 0; k < n; ++k) {
        double l = lam[k];
        for (int it = 0; it < 3; ++it) {
            const double fv = ((l - tr) * l + c1) * l - det;
            const double dv = (3.0 * l - 2.0 * tr) * l + c1;
            if (dv == 0.0 || !isfinite(fv / dv)) break;
            l = l - fv / dv;
        }
        lam[k] = l;
    }
    return n;
}

// unit eigenvector of M for the eigenvalue lam: the largest cross product of two rows of M - lam I
__host__ __device__ bool eigvec3(const double M[3][3], double lam, double v[3])
{
    double A[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A[i][j] = M[i][j] - (i == j ? lam : 0.0);
    double best = -1.0;
    const int pr[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    for (int k = 0; k < 3; ++k) {
        const double* r = A[pr[k][0]];
        const double* s = A[pr[k][1]];
        double w[3] = {r[1] * s[2] - r[2] * s[1], r[2] * s[0] - r[0] * s[2], r[0] * s[1] - r[1] * s[0]};
        const double nn = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
        if (nn > best) { best = nn; v[0] = w[0]; v[1] = w[1]; v[2] = w[2]; }
    }
    if (!(best > 0.0)) return false;
    const double nrm = sqrt(best);
    for (int i = 0; i < 3; ++i) v[i] = v[i] / nrm;
    return true;
}

// x <- (M - lam I)^{-1} x by LU with partial pivoting; a pivot smaller than tiny is taken as tiny, since inverse iteration solves
// with a shift that is an eigenvalue to rounding
__host__ __device__ void shifted_solve(const double M[3][3], double lam, double tiny, double x[3])
{
    double A[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) A[i][j] = M[i][j] - (i == j ? lam : 0.0);
    for (int k = 0; k < 3; ++k) {
        int piv = k;
        for (int i = k + 1; i < 3; ++i)
            if (fabs(A[i][k]) > fabs(A[piv][k])) piv = i;
        if (piv != k) {
            for (int j = 0; j < 3; ++j) { const double t = A[k][j]; A[k][j] = A[piv][j]; A[piv][j] = t; }
            const double t = x[k]; x[k] = x[piv]; x[piv] = t;
        }
        if (fabs(A[k][k]) < tiny) A[k][k] = A[k][k] < 0.0 ? -tiny : tiny;
        for (int i = k + 1; i < 3; ++i) {
            const double l = A[i][k] / A[k][k];
            for (int j = k + 1; j < 3; ++j) A[i][j] = A[i][j] - l * A[k][j];
            x[i] = x[i] - l * x[k];
        }
    }
    for (int i = 2; i >= 0; --i) {
        double t = x[i];
        for (int j = i + 1; j < 3; ++j) t = t - A[i][j] * x[j];
        x[i] = t / A[i][i];
    }
}

// unit eigenvector of M for the eigenvalue nearest lam: three steps of inverse iteration on M itself from the start vector v.  The
// residual of the result is a rounding of |M|, whatever digits the characteristic polynomial lost on lam (LAPACK's eigenvectors
// have the same backward error); false when a step does not give a finite nonzero vector
__host__ __device__ bool inverse_iteration(const double M[3][3], double lam, double tiny, double v[3])
{
    for (int it = 0; it < 3; ++it) {
        double x[3] = {v[0], v[1], v[2]};
        shifted_solve(M, lam, tiny, x);
        const double nn = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
        if (!(nn > 0.0) || !isfinite(nn)) return false;
        for (int i = 0; i < 3; ++i) v[i] = x[i] / nn;
    }
    return true;
}

// the three eigenvectors of M (unit, one per row of V), from eigenvalues that need only be near: the cubic's root of smallest
// magnitude, its eigenvector by inverse iteration, then the other two eigenvalues from the 2 x 2 block that remains after a
// Householder reflection takes that eigenvector to e1; returns how many eigenvectors it found
__host__ __device__ int eig3_vectors(const double M[3][3], double V[3][3])
{
    double nrm = 0.0;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) nrm += M[i][j] * M[i][j];
    nrm = sqrt(nrm);
    if (!(nrm > 0.0) || !isfinite(nrm)) return 0;
    const double tiny = 2.220446049250313e-16 * nrm;
    double lam[3];
    const int nr = eig3_real(M, lam);
    double l0 = lam[0];
    for (int k = 1; k < nr; ++k)
        if (fabs(lam[k]) < fabs(l0)) l0 = lam[k];
    double v[3] = {1.0, 1.0, 1.0};
    if (!eigvec3(M, l0, v)) { v[0] = 1.0; v[1] = 1.0; v[2] = 1.0; }
    if (!inverse_iteration(M, l0, tiny, v)) return 0;
    // B = H M H with H = I - 2 u u^T / u^T u, H v = -+e1: its lower-right 2 x 2 block holds the other two eigenvalues
    double u[3] = {v[0] + (v[0] >= 0.0 ? 1.0 : -1.0), v[1], v[2]};
    const double uu = u[0] * u[0] + u[1] * u[1] + u[2] * u[2];
    double H[3][3], T[3][3], B[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) H[i][j] = (i == j ? 1.0 : 0.0) - 2.0 * u[i] * u[j] / uu;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) T[i][j] = M[i][0] * H[0][j] + M[i][1] * H[1][j] + M[i][2] * H[2][j];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) B[i][j] = H[i][0] * T[0][j] + H[i][1] * T[1][j] + H[i][2] * T[2][j];
    const double p = B[1][1], q = B[1][2], r = B[2][1], s = B[2][2];
    const double half = 0.5 * (p + s), hd = 0.5 * (p - s);
    // the pencil of the direct fit has real eigenvalues: a discriminant that rounding pushed below zero is a double root
    const double sq = sqrt(fmax(hd * hd + q * r, 0.0));
    const double la = half + (half >= 0.0 ? sq : -sq);
    const double lb = la != 0.0 ? (p * s - q * r) / la : half - (half >= 0.0 ? sq : -sq);
    for (int i = 0; i < 3; ++i) V[0][i] = v[i];
    int n = 1;
    const double others[2] = {la, lb};
    for (int k = 0; k < 2; ++k) {
        double w[3] = {1.0, 1.0, 1.0};
        if (!eigvec3(M, others[k], w)) { w[0] = 1.0; w[1] = 1.0; w[2] = 1.0; }
        if (!inverse_iteration(M, others[k], tiny, w)) continue;
        for (int i = 0; i < 3; ++i) V[n][i] = w[i];
        ++n;
    }
    return n;
}

// direct (Halir-Flusser) fit from the 21 scatter sums; S1 = D1^T D1, S2 = D1^T D2, S3 = D2^T D2 with D1 = [x^2, xy, y^2], D2 = [x, y, 1]
__host__ __device__ Fit fit_from_scatter(const double S1[3][3], const double S2[3][3], const double S3[3][3])
{
    Fit r;
    r.status = 0;
    for (int i = 0; i < 5; ++i) r.p[i] = 0.0;
    double iS3[3][3];
    if (!inv3(S3, iS3)) { r.status = -1; return r; }
    double T1[3][3], R[3][3], P[3][3], M[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) T1[i][j] = S2[i][0] * iS3[0][j] + S2[i][1] * iS3[1][j] + S2[i][2] * iS3[2][j];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[i][j] = S1[i][j] - (T1[i][0] * S2[j][0] + T1[i][1] * S2[j][1] + T1[i][2] * S2[j][2]);
    for (int j = 0; j < 3; ++j) { M[0][j] = 0.5 * R[2][j]; M[1][j] = -R[1][j]; M[2][j] = 0.5 * R[0][j]; }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) P[i][j] = -iS3[i][0] * S2[j][0] + -iS3[i][1] * S2[j][1] + -iS3[i][2] * S2[j][2];
    double V[3][3], a1[3];
    const int n = eig3_vectors(M, V);
    int admissible = 0;
    for (int k = 0; k < n; ++k) {
        const double* v = V[k];
        if (4.0 * (v[0] * v[2]) - v[1] * v[1] > 0) {
            ++admissible;
            a1[0] = v[0]; a1[1] = v[1]; a1[2] = v[2];
        }
    }
    if (admissible != 1) return r;
    // the eigenvector's sign is free (LAPACK leaves it to its QR sweeps): take the one that lists the shorter semi-axis first
    conic_params(a1, P, r.p);
    if (r.p[2] > r.p[3]) {
        a1[0] = -a1[0]; a1[1] = -a1[1]; a1[2] = -a1[2];
        conic_params(a1, P, r.p);
    }
    r.status = 1;
    return r;
}

__host__ __device__ __forceinline__ double ell_fun(const double p[5], double ct_, double st_, double t, double xi, double yi)
{
    const double ct = cos(t), st = sin(t);
    const double xt = p[0] + p[2] * ct_ * ct - p[3] * st_ * st;
    const double yt = p[1] + p[2] * st_ * ct + p[3] * ct_ * st;
    return (xi - xt) * (xi - xt) + (yi - yt) * (yi - yt);
}

// distance of (xi, yi) to the ellipse: the stationary point of the squared distance over the ellipse angle reached from
// t0 = atan2(yi - yc, xi - xc) - theta by safeguarded Newton steps (skimage runs scipy leastsq from the same t0)
__host__ __device__ double ell_residual(const double p[5], double ctheta, double stheta, double xi, double yi)
{
    double t = atan2(yi - p[1], xi - p[0]) - p[4];
    double ft = ell_fun(p, ctheta, stheta, t, xi, yi);
    for (int it = 0; it < 64; ++it) {
        const double ct = cos(t), st = sin(t);
        const double ex = p[2] * ctheta * ct - p[3] * stheta * st, ey = p[2] * stheta * ct + p[3] * ctheta * st;
        const double dx = p[0] + ex - xi, dy = p[1] + ey - yi;
        const double xd = -p[2] * ctheta * st - p[3] * stheta * ct, yd = -p[2] * stheta * st + p[3] * ctheta * ct;
        const double g = dx * xd + dy * yd;                            // half the first derivative
        const double h = xd * xd + yd * yd - (dx * ex + dy * ey);      // half the second derivative
        if (g == 0.0) break;
        double step = h > 0 ? -g / h : (g > 0 ? -0.25 : 0.25);
        step = fmax(-0.5, fmin(0.5, step));
        double tn = t + step, fn = ell_fun(p, ctheta, stheta, tn, xi, yi);
        int back = 0;
        while (fn > ft && back < 40) { step *= 0.5; tn = t + step; fn = ell_fun(p, ctheta, stheta, tn, xi, yi); ++back; }
        if (fn > ft) break;
        const bool done = fabs(step) <= 1e-15 * fmax(1.0, fabs(t));
        t = tn; ft = fn;
        if (done) break;
    }
    return sqrt(ft);
}

__global__ void __launch_bounds__(ETHREADS) k_ellipse_trials(
    int T, const int32_t* __restrict__ trial_centre, const int32_t* __restrict__ samp_off, const int32_t* __restrict__ samp_idx,
    const double* __restrict__ params_in, const double* __restrict__ pts, const int32_t* __restrict__ pt_off, double thr,
    const double* __restrict__ sp_pts, const int32_t* __restrict__ sp_lab, const double* __restrict__ lab_term, int N,
    int32_t* __restrict__ ok, double* __restrict__ params_out, int32_t* __restrict__ n_inl, double* __restrict__ crit,
    double* __restrict__ resid_out, const long long* __restrict__ resid_off)
{
    __shared__ double s_p[5];
    __shared__ int s_status;
    __shared__ double s_red[ETHREADS];
    __shared__ int s_cnt[ETHREADS];
    const int t = blockIdx.x, tid = threadIdx.x;
    const int centre = trial_centre[t];
    const double* cp = pts + 2 * (size_t)pt_off[centre];
    const int n = pt_off[centre + 1] - pt_off[centre];

    if (params_in) {
        if (tid < 5) s_p[tid] = params_in[5 * (size_t)t + tid];
        if (tid == 0) s_status = 1;
    } else if (tid < 32) {
        // 21 scatter sums: lane-strided over the samples in their drawn order, then a fixed butterfly.  The samples are taken
        // about their mean: about the origin the sums of x^4 lose the ellipse's digits to its distance from there (8 000 px out,
        // numpy's fit of the same samples misses some ellipses), about the mean they keep them
        double ox = 0.0, oy = 0.0;
        for (int s = samp_off[t] + tid; s < samp_off[t + 1]; s += 32) {
            ox += cp[2 * (size_t)samp_idx[s]];
            oy += cp[2 * (size_t)samp_idx[s] + 1];
        }
        for (int o = 16; o > 0; o >>= 1) {
            ox += __shfl_xor_sync(0xffffffffu, ox, o);
            oy += __shfl_xor_sync(0xffffffffu, oy, o);
        }
        const int n_smp = samp_off[t + 1] - samp_off[t];
        if (n_smp > 0) { ox = ox / n_smp; oy = oy / n_smp; }
        double acc[21];
        for (int k = 0; k < 21; ++k) acc[k] = 0.0;
        for (int s = samp_off[t] + tid; s < samp_off[t + 1]; s += 32) {
            const double x = cp[2 * (size_t)samp_idx[s]] - ox, y = cp[2 * (size_t)samp_idx[s] + 1] - oy;
            const double d1[3] = {x * x, x * y, y * y}, d2[3] = {x, y, 1.0};
            int k = 0;
            for (int i = 0; i < 3; ++i)
                for (int j = i; j < 3; ++j) acc[k++] += d1[i] * d1[j];
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) acc[k++] += d1[i] * d2[j];
            for (int i = 0; i < 3; ++i)
                for (int j = i; j < 3; ++j) acc[k++] += d2[i] * d2[j];
        }
        for (int k = 0; k < 21; ++k)
            for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(0xffffffffu, acc[k], o);
        if (tid == 0) {
            double S1[3][3], S2[3][3], S3[3][3];
            int k = 0;
            for (int i = 0; i < 3; ++i)
                for (int j = i; j < 3; ++j) { S1[i][j] = acc[k]; S1[j][i] = acc[k]; ++k; }
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) S2[i][j] = acc[k++];
            for (int i = 0; i < 3; ++i)
                for (int j = i; j < 3; ++j) { S3[i][j] = acc[k]; S3[j][i] = acc[k]; ++k; }
            const Fit f = fit_from_scatter(S1, S2, S3);
            s_status = f.status;
            for (int i = 0; i < 5; ++i) s_p[i] = f.p[i];
            if (f.status == 1) { s_p[0] = f.p[0] + ox; s_p[1] = f.p[1] + oy; }
        }
    }
    __syncthreads();
    double p[5];
    for (int i = 0; i < 5; ++i) p[i] = s_p[i];
    const int status = s_status;
    if (status != 1) {
        if (tid == 0) {
            ok[t] = status;
            for (int i = 0; i < 5; ++i) params_out[5 * (size_t)t + i] = p[i];
            n_inl[t] = 0;
            crit[t] = 0.0;
        }
        return;
    }

    const double ctheta = cos(p[4]), stheta = sin(p[4]);
    int cnt = 0;
    for (int i = tid; i < n; i += ETHREADS) {
        const double r = ell_residual(p, ctheta, stheta, cp[2 * (size_t)i], cp[2 * (size_t)i + 1]);
        if (resid_out) resid_out[resid_off[t] + i] = r;
        cnt += fabs(r) < thr;
    }
    // criterion (imsegm/ellipse_fitting.py:121-137): the inside test as written there, per-label terms summed in point order
    const double sin_phi = sin(p[4]), cos_phi = cos(p[4]);
    double acc = 0.0;
    for (int j = tid; j < N; j += ETHREADS) {
        const double r = sp_pts[2 * (size_t)j] - p[0], c = sp_pts[2 * (size_t)j + 1] - p[1];
        const double u = (r * cos_phi + c * sin_phi) / p[2], w = (r * sin_phi - c * cos_phi) / p[3];
        if (u * u + w * w <= 1) acc += lab_term[sp_lab[j]];
    }
    s_red[tid] = acc;
    s_cnt[tid] = cnt;
    __syncthreads();
    for (int o = ETHREADS / 2; o > 0; o >>= 1) {
        if (tid < o) { s_red[tid] += s_red[tid + o]; s_cnt[tid] += s_cnt[tid + o]; }
        __syncthreads();
    }
    if (tid == 0) {
        ok[t] = 1;
        for (int i = 0; i < 5; ++i) params_out[5 * (size_t)t + i] = p[i];
        n_inl[t] = s_cnt[0];
        crit[t] = s_red[0];
    }
}

// one ellipse into a mask, and per label: its area and its overlap with the ellipse (shared-memory histograms)
__global__ void k_ellipse_overlap(const int32_t* __restrict__ segm, int H, int W, int n_labels, int r0, int c0, int r1, int c1,
                                  double r_org, double c_org, double r_rad, double c_rad, double sin_a, double cos_a,
                                  uint8_t* __restrict__ mask, unsigned long long* __restrict__ counts)
{
    // [2 * n_labels + 1]: area per label | overlap per label | ellipse area; in shared memory up to ELL_SMEM_LABELS labels, else the
    // global counters directly
    extern __shared__ unsigned int s_hist[];
    const bool smem = n_labels <= ELL_SMEM_LABELS;
    if (smem)
        for (int i = threadIdx.x; i < 2 * n_labels + 1; i += blockDim.x) s_hist[i] = 0;
    __syncthreads();
    const long long npx = (long long)H * W;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < npx; i += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(i / W), x = (int)(i % W);
        bool in = false;
        if (y >= r0 && y <= r1 && x >= c0 && x <= c1) {
            // skimage.draw.ellipse: pixel offsets in the clipped bounding box about the shifted centre
            const double r = (double)(y - r0) - r_org, c = (double)(x - c0) - c_org;
            const double u = (r * cos_a + c * sin_a) / r_rad, w = (r * sin_a - c * cos_a) / c_rad;
            in = (u * u + w * w) < 1;
        }
        mask[i] = in;
        const int l = segm[i];
        if (smem) {
            if (l >= 0 && l < n_labels) {
                atomicAdd(&s_hist[l], 1u);
                if (in) atomicAdd(&s_hist[n_labels + l], 1u);
            }
            if (in) atomicAdd(&s_hist[2 * n_labels], 1u);
        } else {
            if (l >= 0 && l < n_labels) {
                atomicAdd(&counts[l], 1ull);
                if (in) atomicAdd(&counts[n_labels + l], 1ull);
            }
            if (in) atomicAdd(&counts[2 * n_labels], 1ull);
        }
    }
    if (!smem) return;
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * n_labels + 1; i += blockDim.x)
        if (s_hist[i]) atomicAdd(&counts[i], (unsigned long long)s_hist[i]);
}

// grey erosion (op 0, minimum) or dilation (op 1, maximum) of a 0/1 mask over a list of footprint offsets, the border mirrored
// about the edge (scipy.ndimage mode 'reflect')
__global__ void k_binary_morph(const uint8_t* __restrict__ in, int H, int W, const int32_t* __restrict__ offs, int n_offs, int op,
                               uint8_t* __restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)H * W) return;
    const int y = (int)(i / W), x = (int)(i % W);
    uint8_t v = op == 0 ? 1 : 0;
    for (int k = 0; k < n_offs; ++k) {
        const int yy = reflect_index(y + offs[2 * k], H), xx = reflect_index(x + offs[2 * k + 1], W);
        const uint8_t s = in[(size_t)yy * W + xx] != 0;
        v = op == 0 ? (v & s) : (v | s);
    }
    out[i] = v;
}

}  // namespace

extern "C" int isb_ellipse_ransac(int T, const int32_t* trial_centre, const int32_t* samp_off, const int32_t* samp_idx, const double* params_in,
                                  int C, const double* pts, const int32_t* pt_off, double thr, const double* sp_pts, const int32_t* sp_lab,
                                  const double* lab_term, int N, int32_t* ok, double* params_out, int32_t* n_inl, double* crit,
                                  double* resid_out, const long long* resid_off, isb_stream_t stream)
{
    ISB_REQUIRE(T > 0 && C > 0 && N >= 0, "T and C must be positive and N non-negative");
    ISB_REQUIRE(trial_centre && pts && pt_off && ok && params_out && n_inl && crit, "null pointer");
    ISB_REQUIRE(params_in || (samp_off && samp_idx), "either params_in or the sample table (samp_off, samp_idx) is required");
    ISB_REQUIRE(N == 0 || (sp_pts && sp_lab && lab_term), "null superpixel points, labels or label terms with N > 0");
    ISB_REQUIRE(!resid_out || resid_off, "resid_out needs resid_off");
    k_ellipse_trials<<<T, ETHREADS, 0, (cudaStream_t)stream>>>(T, trial_centre, samp_off, samp_idx, params_in, pts, pt_off, thr, sp_pts, sp_lab,
                                                                lab_term, N, ok, params_out, n_inl, crit, resid_out, resid_off);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_ellipse_overlap(const int32_t* segm, int H, int W, int n_labels, const int32_t* bbox_host, const double* geom_host,
                                   uint8_t* mask, unsigned long long* counts, isb_stream_t stream)
{
    ISB_REQUIRE(segm && bbox_host && geom_host && mask && counts, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0, "H and W must be positive");
    ISB_REQUIRE(n_labels > 0, "n_labels must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    ISB_CUDA_CHECK(cudaMemsetAsync(counts, 0, (2 * (size_t)n_labels + 1) * sizeof(unsigned long long), st));
    const long long npx = (long long)H * W;
    const int blocks = (int)min((npx + 255) / 256, 132LL * 8);
    const size_t smem = n_labels <= ELL_SMEM_LABELS ? (2 * (size_t)n_labels + 1) * sizeof(unsigned int) : 0;
    k_ellipse_overlap<<<blocks, 256, smem, st>>>(
        segm, H, W, n_labels, bbox_host[0], bbox_host[1], bbox_host[2], bbox_host[3], geom_host[0], geom_host[1], geom_host[2],
        geom_host[3], geom_host[4], geom_host[5], mask, counts);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}

extern "C" int isb_binary_morph_footprint(const uint8_t* in, int H, int W, const int32_t* offsets, int n_offsets, int op, uint8_t* out,
                                          isb_stream_t stream)
{
    ISB_REQUIRE(in && offsets && out, "null pointer");
    ISB_REQUIRE(H > 0 && W > 0 && n_offsets > 0, "H, W and n_offsets must be positive");
    ISB_REQUIRE(op == 0 || op == 1, "op must be 0 or 1");
    ISB_REQUIRE(in != out, "in and out must differ");
    const long long npx = (long long)H * W;
    k_binary_morph<<<(unsigned)((npx + 255) / 256), 256, 0, (cudaStream_t)stream>>>(in, H, W, offsets, n_offsets, op, out);
    ISB_LAUNCH_CHECK();
    return ISB_OK;
}
