// oracle/fundamental.cpp -- TEST INFRASTRUCTURE ONLY (see oracle/sgs_oracle.cpp header): CPU restatement of
//   cv::findFundamentalMat(points1, points2, cv::FM_RANSAC, 1.0, 0.99)      as called at src/Frame.cc:469-472
// together with the point selection in front of it (src/Frame.cc:454-468).
//
// OpenCV is a third-party dependency that is not vendored under /root/reference (the reference pins 3.4.15, README.md:91).  The
// algorithm below restates calib3d/fundam.cpp + calib3d/ptsetreg.cpp + core/lapack.cpp (JacobiSVD) + core/mathfuncs.cpp
// (solveCubic) and is PINNED against cv2 4.13 run in the build container (tests/golden/make_golden_fm.py ->
// tests/golden/fm_ransac.npz): F agrees to ~1e-12 and the inlier masks are identical.  Behaviour that defines the result:
//   * RNG rng((uint64)-1), MWC generator x = (uint32)x * 4164903690 + (x >> 32); uniform(0, n) = next() % n
//   * 7 distinct indices per iteration, redrawn while the LAST point is collinear with two earlier ones: at most 10000 attempts in
//     RANSAC, which passes that cap to getSubset, and getSubset's default of 1000 in LMedS; a failed first draw returns no matrix
//   * the 7-point solver normalises the 7 points (centroid, mean distance sqrt 2) [4.13 behaviour, found by probe], takes the two
//     missing right singular vectors from JacobiSVD's completion step (fixed RNG(0x12345678) sign vectors projected off the row
//     space), solves det(l f1 + (1 - l) f2) = 0 with cv::solveCubic, and scales each F to F33 = 1
//   * error = (float)max(d1^2/(a1^2+b1^2), d2^2/(a2^2+b2^2)) in double, inlier iff <= (float)(thr*thr)
//   * a model replaces the best one iff inliers > max(best, 6); niters = RANSACUpdateNumIters(...) after every improvement
//   * no refit on the inliers; fewer than 15 pairs never reach RANSAC: 8..14 -> LMedS, exactly 7 -> the 7-point solver itself, fewer -> empty (all restated below)
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#define SGO_API extern "C" __attribute__((visibility("default")))

namespace {

struct CvRng {
    uint64_t state;
    explicit CvRng(uint64_t s) : state(s) {}
    inline unsigned next() { state = (uint64_t)(unsigned)state * 4164903690U + (unsigned)(state >> 32); return (unsigned)state; }
    inline int uniform(int a, int b) { return a == b ? a : (int)(next() % (unsigned)(b - a) + a); }
};

// core/lapack.cpp JacobiSVDImpl_<double>: one-sided Jacobi on the n rows (length m) of At; rows come out as sigma_i * u_i sorted by
// decreasing sigma; rows n..n1-1 are completed from fixed pseudo-random sign vectors (see header).  Vt is not needed here.
void jacobi_rows(double* At, int m, int n, int n1, double* W) {
    const double eps = DBL_EPSILON * 10, minval = DBL_MIN;
    const int max_iter = std::max(m, 30);
    for (int i = 0; i < n; i++) { double sd = 0; for (int k = 0; k < m; k++) sd += At[i * m + k] * At[i * m + k]; W[i] = sd; }
    for (int iter = 0; iter < max_iter; iter++) {
        bool changed = false;
        for (int i = 0; i < n - 1; i++)
            for (int j = i + 1; j < n; j++) {
                double* Ai = At + i * m; double* Aj = At + j * m;
                double a = W[i], p = 0, b = W[j];
                for (int k = 0; k < m; k++) p += Ai[k] * Aj[k];
                if (std::abs(p) <= eps * std::sqrt(a * b)) continue;
                p *= 2;
                const double beta = a - b, gamma = hypot(p, beta);
                double c, s;
                if (beta < 0) { const double delta = (gamma - beta) * 0.5; s = std::sqrt(delta / gamma); c = p / (gamma * s * 2); }
                else { c = std::sqrt((gamma + beta) / (gamma * 2)); s = p / (gamma * c * 2); }
                a = b = 0;
                for (int k = 0; k < m; k++) {
                    const double t0 = c * Ai[k] + s * Aj[k], t1 = -s * Ai[k] + c * Aj[k];
                    Ai[k] = t0; Aj[k] = t1;
                    a += t0 * t0; b += t1 * t1;
                }
                W[i] = a; W[j] = b;
                changed = true;
            }
        if (!changed) break;
    }
    for (int i = 0; i < n; i++) { double sd = 0; for (int k = 0; k < m; k++) sd += At[i * m + k] * At[i * m + k]; W[i] = std::sqrt(sd); }
    for (int i = 0; i < n - 1; i++) {
        int j = i;
        for (int k = i + 1; k < n; k++) if (W[j] < W[k]) j = k;
        if (i != j) { std::swap(W[i], W[j]); for (int k = 0; k < m; k++) std::swap(At[i * m + k], At[j * m + k]); }
    }
    CvRng rng(0x12345678);
    for (int i = 0; i < n1; i++) {
        double sd = i < n ? W[i] : 0;
        for (int ii = 0; ii < 100 && sd <= minval; ii++) {
            const double val0 = 1. / m;
            for (int k = 0; k < m; k++) At[i * m + k] = (rng.next() & 256) != 0 ? val0 : -val0;
            for (int iter = 0; iter < 2; iter++)
                for (int j = 0; j < i; j++) {
                    sd = 0;
                    for (int k = 0; k < m; k++) sd += At[i * m + k] * At[j * m + k];
                    double asum = 0;
                    for (int k = 0; k < m; k++) { const double t = At[i * m + k] - sd * At[j * m + k]; At[i * m + k] = t; asum += std::abs(t); }
                    asum = asum > eps * 100 ? 1 / asum : 0;
                    for (int k = 0; k < m; k++) At[i * m + k] *= asum;
                }
            sd = 0;
            for (int k = 0; k < m; k++) sd += At[i * m + k] * At[i * m + k];
            sd = std::sqrt(sd);
        }
        const double s = sd > minval ? 1 / sd : 0.;
        for (int k = 0; k < m; k++) At[i * m + k] *= s;
    }
}

// core/mathfuncs.cpp cv::solveCubic for a 4-coefficient polynomial c[0] x^3 + c[1] x^2 + c[2] x + c[3]
int solve_cubic(const double* c, double* r) {
    double a0 = c[0], a1 = c[1], a2 = c[2], a3 = c[3];
    double x0 = 0, x1 = 0, x2 = 0;
    int n = 0;
    if (a0 == 0) {
        if (a1 == 0) {
            if (a2 == 0) n = a3 == 0 ? -1 : 0;
            else { x0 = -a3 / a2; n = 1; }
        } else {
            double d = a2 * a2 - 4 * a1 * a3;
            if (d >= 0) {
                d = std::sqrt(d);
                const double q1 = (-a2 + d) * 0.5, q2 = (a2 + d) * -0.5;
                if (std::fabs(q1) > std::fabs(q2)) { x0 = q1 / a1; x1 = a3 / q1; }
                else { x0 = q2 / a1; x1 = a3 / q2; }
                n = d > 0 ? 2 : 1;
            }
        }
    } else {
        a0 = 1. / a0; a1 *= a0; a2 *= a0; a3 *= a0;
        const double Q = (a1 * a1 - 3 * a2) * (1. / 9);
        const double R = (2 * a1 * a1 * a1 - 9 * a1 * a2 + 27 * a3) * (1. / 54);
        const double Qcubed = Q * Q * Q;
        double d = Qcubed - R * R;
        if (d > 0) {
            const double theta = std::acos(R / std::sqrt(Qcubed)), sqrtQ = std::sqrt(Q);
            const double t0 = -2 * sqrtQ, t1 = theta * (1. / 3), t2 = a1 * (1. / 3);
            x0 = t0 * std::cos(t1) - t2;
            x1 = t0 * std::cos(t1 + (2. * M_PI / 3)) - t2;
            x2 = t0 * std::cos(t1 + (4. * M_PI / 3)) - t2;
            n = 3;
        } else if (d == 0) {
            if (R >= 0) { x0 = -2 * std::pow(R, 1. / 3) - a1 / 3; x1 = std::pow(R, 1. / 3) - a1 / 3; }
            else { x0 = 2 * std::pow(-R, 1. / 3) - a1 / 3; x1 = -std::pow(-R, 1. / 3) - a1 / 3; }
            x2 = 0;
            n = x0 == x1 ? 1 : 2;
            x1 = x0 == x1 ? 0 : x1;
        } else {
            d = std::sqrt(-d);
            double e = std::pow(d + std::fabs(R), 1. / 3);
            if (R > 0) e = -e;
            x0 = (e + Q / e) - a1 * (1. / 3);
            n = 1;
        }
    }
    r[0] = x0; r[1] = x1; r[2] = x2;
    return n;
}

// fundam.cpp run7Point (cv2 4.13: on normalised coordinates).  F: up to 3 row-major 3x3.
int run7point(const float* m1, const float* m2, double* F) {
    double c1x = 0, c1y = 0, c2x = 0, c2y = 0;
    for (int i = 0; i < 7; i++) { c1x += m1[2 * i]; c1y += m1[2 * i + 1]; c2x += m2[2 * i]; c2y += m2[2 * i + 1]; }
    const double t = 1. / 7;
    c1x *= t; c1y *= t; c2x *= t; c2y *= t;
    double s1 = 0, s2 = 0;
    for (int i = 0; i < 7; i++) {
        s1 += std::sqrt((m1[2 * i] - c1x) * (m1[2 * i] - c1x) + (m1[2 * i + 1] - c1y) * (m1[2 * i + 1] - c1y));
        s2 += std::sqrt((m2[2 * i] - c2x) * (m2[2 * i] - c2x) + (m2[2 * i + 1] - c2y) * (m2[2 * i + 1] - c2y));
    }
    s1 *= t; s2 *= t;
    if (s1 < FLT_EPSILON || s2 < FLT_EPSILON) return 0;
    s1 = std::sqrt(2.) / s1; s2 = std::sqrt(2.) / s2;
    double a[9 * 9], w[9];
    std::memset(a, 0, sizeof(a));
    for (int i = 0; i < 7; i++) {
        const double x0 = (m1[2 * i] - c1x) * s1, y0 = (m1[2 * i + 1] - c1y) * s1;
        const double x1 = (m2[2 * i] - c2x) * s2, y1 = (m2[2 * i + 1] - c2y) * s2;
        double* r = a + i * 9;
        r[0] = x1 * x0; r[1] = x1 * y0; r[2] = x1; r[3] = y1 * x0; r[4] = y1 * y0; r[5] = y1; r[6] = x0; r[7] = y0; r[8] = 1;
    }
    jacobi_rows(a, 9, 7, 9, w);
    double* f1 = a + 7 * 9; double* f2 = a + 8 * 9;
    for (int i = 0; i < 9; i++) f1[i] -= f2[i];
    double c[4], r[3] = {0, 0, 0};
    double t0 = f2[4] * f2[8] - f2[5] * f2[7], t1 = f2[3] * f2[8] - f2[5] * f2[6], t2 = f2[3] * f2[7] - f2[4] * f2[6];
    c[3] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2;
    c[2] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2 - f1[3] * (f2[1] * f2[8] - f2[2] * f2[7]) + f1[4] * (f2[0] * f2[8] - f2[2] * f2[6]) -
           f1[5] * (f2[0] * f2[7] - f2[1] * f2[6]) + f1[6] * (f2[1] * f2[5] - f2[2] * f2[4]) - f1[7] * (f2[0] * f2[5] - f2[2] * f2[3]) +
           f1[8] * (f2[0] * f2[4] - f2[1] * f2[3]);
    t0 = f1[4] * f1[8] - f1[5] * f1[7]; t1 = f1[3] * f1[8] - f1[5] * f1[6]; t2 = f1[3] * f1[7] - f1[4] * f1[6];
    c[0] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2;
    c[1] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2 - f2[3] * (f1[1] * f1[8] - f1[2] * f1[7]) + f2[4] * (f1[0] * f1[8] - f1[2] * f1[6]) -
           f2[5] * (f1[0] * f1[7] - f1[1] * f1[6]) + f2[6] * (f1[1] * f1[5] - f1[2] * f1[4]) - f2[7] * (f1[0] * f1[5] - f1[2] * f1[3]) +
           f2[8] * (f1[0] * f1[4] - f1[1] * f1[3]);
    const int n = solve_cubic(c, r);
    if (n < 1 || n > 3) return n < 0 ? 0 : n;
    // T2^T F0 T1 with T = [s 0 -s cx; 0 s -s cy; 0 0 1]
    for (int k = 0; k < n; k++) {
        double lambda = r[k], mu = 1.;
        const double s = f1[8] * r[k] + f2[8];
        double f0[9];
        if (std::fabs(s) > DBL_EPSILON) { mu = 1. / s; lambda *= mu; f0[8] = 1.; } else f0[8] = 0.;
        for (int i = 0; i < 8; i++) f0[i] = f1[i] * lambda + f2[i] * mu;
        const double T1[9] = {s1, 0, -s1 * c1x, 0, s1, -s1 * c1y, 0, 0, 1}, T2[9] = {s2, 0, -s2 * c2x, 0, s2, -s2 * c2y, 0, 0, 1};
        double tmp[9], out[9];
        for (int i = 0; i < 3; i++)       // tmp = T2^T * f0
            for (int j = 0; j < 3; j++) { double v = 0; for (int q = 0; q < 3; q++) v += T2[q * 3 + i] * f0[q * 3 + j]; tmp[i * 3 + j] = v; }
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) { double v = 0; for (int q = 0; q < 3; q++) v += tmp[i * 3 + q] * T1[q * 3 + j]; out[i * 3 + j] = v; }
        if (std::fabs(out[8]) > DBL_EPSILON) { const double sc = 1. / out[8]; for (int i = 0; i < 9; i++) out[i] *= sc; }
        std::memcpy(F + 9 * k, out, sizeof(out));
    }
    return n;
}

bool have_collinear(const float* m, int count) {      // fundam.cpp haveCollinearPoints: only the last point is tested
    const int i = count - 1;
    for (int j = 0; j < i; j++) {
        const double dx1 = m[2 * j] - m[2 * i], dy1 = m[2 * j + 1] - m[2 * i + 1];
        for (int k = 0; k < j; k++) {
            const double dx2 = m[2 * k] - m[2 * i], dy2 = m[2 * k + 1] - m[2 * i + 1];
            if (std::fabs(dx2 * dy1 - dy2 * dx1) <= FLT_EPSILON * (std::fabs(dx1) + std::fabs(dy1) + std::fabs(dx2) + std::fabs(dy2))) return true;
        }
    }
    return false;
}

void compute_errors(const float* m1, const float* m2, int n, const double* F, float* err) {      // FMEstimatorCallback::computeError
    for (int i = 0; i < n; i++) {
        const double x1 = m1[2 * i], y1 = m1[2 * i + 1], x2 = m2[2 * i], y2 = m2[2 * i + 1];
        double a = F[0] * x1 + F[1] * y1 + F[2], b = F[3] * x1 + F[4] * y1 + F[5], c = F[6] * x1 + F[7] * y1 + F[8];
        const double s2 = 1. / (a * a + b * b), d2 = x2 * a + y2 * b + c;
        a = F[0] * x2 + F[3] * y2 + F[6]; b = F[1] * x2 + F[4] * y2 + F[7]; c = F[2] * x2 + F[5] * y2 + F[8];
        const double s1 = 1. / (a * a + b * b), d1 = x1 * a + y1 * b + c;
        err[i] = (float)std::max(d1 * d1 * s1, d2 * d2 * s2);
    }
}

int find_inliers(const float* m1, const float* m2, int n, const double* F, float t, uint8_t* mask) {
    int nz = 0;
    for (int i = 0; i < n; i++) {
        const double x1 = m1[2 * i], y1 = m1[2 * i + 1], x2 = m2[2 * i], y2 = m2[2 * i + 1];
        double a = F[0] * x1 + F[1] * y1 + F[2], b = F[3] * x1 + F[4] * y1 + F[5], c = F[6] * x1 + F[7] * y1 + F[8];
        const double s2 = 1. / (a * a + b * b), d2 = x2 * a + y2 * b + c;
        a = F[0] * x2 + F[3] * y2 + F[6]; b = F[1] * x2 + F[4] * y2 + F[7]; c = F[2] * x2 + F[5] * y2 + F[8];
        const double s1 = 1. / (a * a + b * b), d1 = x1 * a + y1 * b + c;
        const float err = (float)std::max(d1 * d1 * s1, d2 * d2 * s2);
        const int f = err <= t;
        mask[i] = (uint8_t)f; nz += f;
    }
    return nz;
}

int update_num_iters(double p, double ep, int model_points, int max_iters) {      // ptsetreg.cpp RANSACUpdateNumIters
    p = std::min(std::max(p, 0.), 1.); ep = std::min(std::max(ep, 0.), 1.);
    double num = std::max(1. - p, DBL_MIN), denom = 1. - std::pow(1. - ep, model_points);
    if (denom < DBL_MIN) return 0;
    num = std::log(num); denom = std::log(denom);
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int)std::nearbyint(num / denom);
}

}  // namespace

SGO_API int sgo_run7point(const float* m1, const float* m2, double* F27) { return run7point(m1, m2, F27); }

// info (may be NULL): [0] iterations run, [1] inliers of the returned model, [2] final niters
SGO_API int sgo_find_fundamental_ransac(const float* m1, const float* m2, int n, double thresh, double confidence, int max_iters, double* F,
                                        uint8_t* mask_out, int32_t* info) {
    if (info) info[0] = info[1] = info[2] = 0;
    if (thresh <= 0) thresh = 3;
    if (confidence < DBL_EPSILON || confidence > 1 - DBL_EPSILON) confidence = 0.99;
    if (n < 15) {
        // fundam.cpp cv::findFundamentalMat: fewer than 15 pairs never reach RANSAC.  < 7: empty; == 7: the 7-point solver directly (up to three
        // stacked solutions; the first is returned); 8..14: LMeDSPointSetRegistrator(cb, 7, confidence, max_iters).run (ptsetreg.cpp): a fixed
        // number of samples, max(RANSACUpdateNumIters(confidence, 0.45, 7, max_iters), 3), each drawn in at most 1000 attempts (getSubset's
        // default; RANSAC passes 10000), the model with the smallest median error (element count/2 of the sorted errors), inliers within
        // sigma = 2.5 * 1.4826 * (1 + 5 / (count - 7)) * sqrt(median); the result is dropped when fewer than 7 pairs are inliers.
        if (n < 7) return 0;
        if (n == 7) {             // runKernel directly: the stacked solutions; callers read rows 0..2 = the first one (src/Frame.cc:617-619)
            double models7[27];
            const int nm = run7point(m1, m2, models7);
            if (nm <= 0) return 0;
            std::memcpy(F, models7, 9 * sizeof(double));
            if (mask_out) std::memset(mask_out, 1, n);
            if (info) { info[0] = 1; info[1] = 7; info[2] = 1; }
            return 1;
        }
        CvRng rng((uint64_t)-1);
        const int niters = std::max(update_num_iters(confidence, 0.45, 7, max_iters), 3);
        double min_median = DBL_MAX, best[9], models[27];
        float ms1[14], ms2[14];
        std::vector<float> err(n);
        int iter = 0;
        for (iter = 0; iter < niters; iter++) {
            bool found = false;
            for (int attempt = 0; attempt < 1000 && !found; attempt++) {
                int idx[7];
                for (int i = 0; i < 7; i++) {
                    int v;
                    for (v = rng.uniform(0, n); std::find(idx, idx + i, v) != idx + i; v = rng.uniform(0, n)) {}
                    idx[i] = v;
                    ms1[2 * i] = m1[2 * v]; ms1[2 * i + 1] = m1[2 * v + 1]; ms2[2 * i] = m2[2 * v]; ms2[2 * i + 1] = m2[2 * v + 1];
                }
                found = !have_collinear(ms1, 7) && !have_collinear(ms2, 7);
            }
            if (!found) { if (iter == 0) return 0; break; }
            const int nmodels = run7point(ms1, ms2, models);
            for (int k = 0; k < nmodels; k++) {
                compute_errors(m1, m2, n, models + 9 * k, err.data());
                std::nth_element(err.begin(), err.begin() + n / 2, err.end());
                const double median = err[n / 2];
                if (median < min_median) { min_median = median; std::memcpy(best, models + 9 * k, sizeof(best)); }
            }
        }
        if (!(min_median < DBL_MAX)) return 0;
        double sigma = 2.5 * 1.4826 * (1 + 5. / (n - 7)) * std::sqrt(min_median);
        sigma = std::max(sigma, 0.001);
        std::vector<uint8_t> mask(n);
        const int good = find_inliers(m1, m2, n, best, (float)(sigma * sigma), mask.data());
        if (info) { info[0] = iter; info[1] = good; info[2] = niters; }
        if (good < 7) return 0;
        std::memcpy(F, best, sizeof(best));
        if (mask_out) std::memcpy(mask_out, mask.data(), n);
        return 1;
    }
    CvRng rng((uint64_t)-1);
    int niters = std::max(max_iters, 1), max_good = 0, iter = 0;
    const float t = (float)(thresh * thresh);
    std::vector<uint8_t> mask(n), best_mask(n);
    double best[9], models[27];
    float ms1[14], ms2[14];
    for (iter = 0; iter < niters; iter++) {
        bool found = false;
        for (int attempt = 0; attempt < 10000 && !found; attempt++) {
            int idx[7];
            for (int i = 0; i < 7; i++) {
                int v;
                for (v = rng.uniform(0, n); std::find(idx, idx + i, v) != idx + i; v = rng.uniform(0, n)) {}
                idx[i] = v;
                ms1[2 * i] = m1[2 * v]; ms1[2 * i + 1] = m1[2 * v + 1]; ms2[2 * i] = m2[2 * v]; ms2[2 * i + 1] = m2[2 * v + 1];
            }
            found = !have_collinear(ms1, 7) && !have_collinear(ms2, 7);
        }
        if (!found) { if (iter == 0) return 0; break; }
        const int nmodels = run7point(ms1, ms2, models);
        if (nmodels <= 0) continue;
        for (int k = 0; k < nmodels; k++) {
            const int good = find_inliers(m1, m2, n, models + 9 * k, t, mask.data());
            if (good > std::max(max_good, 6)) {
                std::swap(mask, best_mask);
                std::memcpy(best, models + 9 * k, sizeof(best));
                max_good = good;
                niters = update_num_iters(confidence, (double)(n - good) / n, 7, niters);
            }
        }
    }
    if (info) { info[0] = iter; info[1] = max_good; info[2] = niters; }
    if (max_good <= 0) return 0;
    std::memcpy(F, best, sizeof(best));
    if (mask_out) std::memcpy(mask_out, best_mask.data(), n);
    return 1;
}

// src/Frame.cc:454-472: pairs whose PREVIOUS point lies outside the previous frame's dynamic boxes feed the estimator when the
// previous frame had such boxes and more than 20 pairs survive; otherwise all pairs do.  boxes: x, y, w, h floats.
// Returns the number of pairs written to sel1 / sel2 (cap n each).
SGO_API int sgo_select_static_pairs(const float* cur, const float* prev, int n, const float* boxes, int nboxes, int prev_have_dyn, float* sel1, float* sel2) {
    int cnt = 0;
    if (prev_have_dyn) {
        for (int i = 0; i < n; i++) {
            const float x = prev[2 * i], y = prev[2 * i + 1];
            bool in = false;
            for (int b = 0; b < nboxes && !in; b++) {
                const float* r = boxes + 4 * b;
                in = x > r[0] && x < r[0] + r[2] && y > r[1] && y < r[1] + r[3];
            }
            if (!in) { sel1[2 * cnt] = cur[2 * i]; sel1[2 * cnt + 1] = cur[2 * i + 1]; sel2[2 * cnt] = x; sel2[2 * cnt + 1] = y; cnt++; }
        }
        if (cnt > 20) return cnt;
    }
    std::memcpy(sel1, cur, sizeof(float) * 2 * n); std::memcpy(sel2, prev, sizeof(float) * 2 * n);
    return n;
}
