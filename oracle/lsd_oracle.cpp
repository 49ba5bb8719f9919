/*
 * oracle/lsd_oracle.cpp -- CPU ORACLE for the LSD flavour of line_lbd_detect.  TEST INFRASTRUCTURE ONLY.
 *
 * Restates, without OpenCV:
 *   line_lbd/class/line_lbd_allclass.cpp:26-36,125-148,200-221   (detect_filter_lines, filter_lines, keylines_to_mat)
 *   line_lbd/libs/LSDDetector.cpp:55-101,153-256                 (one-octave pyramid, KeyLine fill, 10-px border rejection)
 *   line_lbd/libs/lsd.cpp:80-158,414-1154                        (LineSegmentDetectorImpl, LSD_REFINE_ADV, default parameters:
 *                                                                 scale 0.8, sigma_scale 0.6, quant 2, ang_th 22.5, log_eps 0,
 *                                                                 density_th 0.7, n_bins 1024 -- LSDDetector.cpp:173 ignores LSDOptions)
 * including the vendored quirks (rect_nfa's tailp->p.x-for-p.y slip and integer step slopes, lsd.cpp:1057-1065).
 * OpenCV calls inside (GaussianBlur 7x7 sigma 0.6/0.8 on CV_64F, resize INTER_LINEAR x0.8 on CV_64F, fastAtan2, cvtColor) are
 * restated from OpenCV's algorithms and pinned against the in-container cv2 4.13 (tests/test_oracle_lines.py).
 * The Gaussian kernel is cv2 4.13's bit-exact getGaussianKernel(7, 0.6 / 0.8) (sigma = 0.7499999999999999, lsd.cpp:453) (it differs from exp()-based kernels in the last ulp).
 *
 * The seed list is visited in RASTER order: flsd walks its coorlist vector by index (lsd.cpp:478-480), the gradient-bin links that ll_angle
 * also builds (lsd.cpp:588-634) are never followed.
 *
 * PARITY: PINNED to the reference.  (1) The reference's own lsd.cpp, compiled from /root/reference into oracle/_ref/liblsd_ref.so
 * (oracle/ref/lsd_ref.cpp, oracle/Makefile target `ref`), returns byte-identical raw segments on every fixture, synthetic and
 * degenerate image tried (tests/test_oracle_ref_lsd.py); its segment counts and checksums are recorded in the committed goldens, so the
 * pin also holds where the reference is absent (tests/test_goldens_sequence.py).  (2) The one LSD output the reference ships
 * (detect_3d_cuboid/data/edge_detection/LSD/0000_edge.txt) is reproduced whole: 271 of 271 segments, in order, to its six significant
 * digits (tests/test_oracle_lines.py).  The OpenCV primitives inside are pinned against cv2 4.13.
 */
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "orc_api.h"

extern "C" void orc_bgr2gray(const uint8_t *bgr, int w, int h, int stride, uint8_t *gray, int gstride, int fixed15);

namespace {

const double kPI = 3.1415926535897932384626433832795; /* CV_PI */
const double kNOTDEF = -1024.0;
const double kDegToRads = kPI / 180;
const double kM_3_2_PI = (3 * kPI) / 2;
const double kM_2__PI = (2 * kPI);
const double kLN10 = 2.30258509299404568402;

/* cv::fastAtan2 (OpenCV core/mathfuncs_core: atan_f32), degrees */
inline float fast_atan2(float y, float x)
{
    const float p1 = 0.9997878412794807f * (float)(180 / kPI);
    const float p3 = -0.3258083974640975f * (float)(180 / kPI);
    const float p5 = 0.1555786518463281f * (float)(180 / kPI);
    const float p7 = -0.04432655554792128f * (float)(180 / kPI);
    const float ax = std::abs(x), ay = std::abs(y);
    float a, c, c2;
    if (ax >= ay) {
        c = ay / (ax + (float)DBL_EPSILON);
        c2 = c * c;
        a = (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    } else {
        c = ax / (ay + (float)DBL_EPSILON);
        c2 = c * c;
        a = 90.f - (((p7 * c2 + p5) * c2 + p3) * c2 + p1) * c;
    }
    if (x < 0) a = 180.f - a;
    if (y < 0) a = 360.f - a;
    return a;
}

inline int reflect101(int p, int n)
{
    if (n == 1) return 0;
    while (p < 0 || p >= n) p = (p < 0) ? -p : 2 * n - 2 - p;
    return p;
}

/* cv::GaussianBlur(CV_64F, 7x7, sigma 0.6/0.8, BORDER_REFLECT_101): row filter (k = 0..6 in order), then the symmetric column
 * filter (centre tap first, then ky[k] * (below + above)) -- the operation order of OpenCV's generic C paths */
const double kGauss7[7] = {0x1.763496d347532p-13, 0x1.f1e23259cfdc1p-7, 0x1.bfd7fac1bd5a8p-3, 0x1.10562a79786afp-1,
                           0x1.bfd7fac1bd5a8p-3, 0x1.f1e23259cfdc1p-7, 0x1.763496d347532p-13};

void gaussian_blur7(const std::vector<double> &src, int w, int h, std::vector<double> &dst)
{
    std::vector<double> tmp((size_t)w * h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            double s = kGauss7[0] * src[(size_t)y * w + reflect101(x - 3, w)];
            for (int k = 1; k < 7; k++) s += kGauss7[k] * src[(size_t)y * w + reflect101(x + k - 3, w)];
            tmp[(size_t)y * w + x] = s;
        }
    dst.resize((size_t)w * h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            double s = kGauss7[3] * tmp[(size_t)y * w + x];
            for (int k = 1; k <= 3; k++) s += kGauss7[3 + k] * (tmp[(size_t)reflect101(y + k, h) * w + x] + tmp[(size_t)reflect101(y - k, h) * w + x]);
            dst[(size_t)y * w + x] = s;
        }
}

/* cv::resize(CV_64F, fx = fy = scale, INTER_LINEAR): float coefficients, double accumulation, horizontal then vertical */
void resize_linear(const std::vector<double> &src, int sw, int sh, double scale, std::vector<double> &dst, int &dw, int &dh)
{
    dw = (int)std::lrint(sw * scale);
    dh = (int)std::lrint(sh * scale);
    const double inv_x = 1. / scale, inv_y = 1. / scale;
    std::vector<int> xofs(dw), yofs(dh);
    std::vector<float> ax(2 * (size_t)dw), ay(2 * (size_t)dh);
    int xmax = dw;
    for (int dx = 0; dx < dw; dx++) {
        float fx = (float)((dx + 0.5) * inv_x - 0.5);
        int sx = (int)std::floor(fx);
        fx -= sx;
        if (sx < 0) {
            fx = 0;
            sx = 0;
        }
        if (sx + 1 >= sw) {
            xmax = std::min(xmax, dx);
            if (sx >= sw - 1) {
                fx = 0;
                sx = sw - 1;
            }
        }
        xofs[dx] = sx;
        ax[2 * dx] = 1.f - fx;
        ax[2 * dx + 1] = fx;
    }
    for (int dy = 0; dy < dh; dy++) {
        float fy = (float)((dy + 0.5) * inv_y - 0.5);
        int sy = (int)std::floor(fy);
        fy -= sy;
        yofs[dy] = sy;
        ay[2 * dy] = 1.f - fy;
        ay[2 * dy + 1] = fy;
    }
    auto clip = [](int x, int a, int b) { return x >= a ? (x < b ? x : b - 1) : a; };
    dst.resize((size_t)dw * dh);
    std::vector<double> r0(dw), r1(dw);
    auto hrow = [&](int sy, std::vector<double> &out) {
        const double *S = &src[(size_t)sy * sw];
        for (int dx = 0; dx < dw; dx++) {
            if (dx < xmax)
                out[dx] = S[xofs[dx]] * ax[2 * dx] + S[xofs[dx] + 1] * ax[2 * dx + 1];
            else
                out[dx] = S[xofs[dx]] * 1.0;
        }
    };
    for (int dy = 0; dy < dh; dy++) {
        hrow(clip(yofs[dy], 0, sh), r0);
        hrow(clip(yofs[dy] + 1, 0, sh), r1);
        const float b0 = ay[2 * dy], b1 = ay[2 * dy + 1];
        for (int dx = 0; dx < dw; dx++) dst[(size_t)dy * dw + dx] = r0[dx] * b0 + r1[dx] * b1;
    }
}

/* -------------------------------------------------------------------------------- lsd.cpp helpers (:80-158) */
inline double dist_sq(double x1, double y1, double x2, double y2) { return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1); }
inline double dist2(double x1, double y1, double x2, double y2) { return std::sqrt(dist_sq(x1, y1, x2, y2)); }
inline double angle_diff_signed(double a, double b)
{
    double diff = a - b;
    while (diff <= -kPI) diff += kM_2__PI;
    while (diff > kPI) diff -= kM_2__PI;
    return diff;
}
inline double angle_diff(double a, double b) { return std::fabs(angle_diff_signed(a, b)); }
inline bool double_equal(double a, double b)
{
    if (a == b) return true;
    const double abs_diff = std::fabs(a - b);
    const double aa = std::fabs(a), bb = std::fabs(b);
    double abs_max = (aa > bb) ? aa : bb;
    if (abs_max < DBL_MIN) abs_max = DBL_MIN;
    return (abs_diff / abs_max) <= (100.0 * DBL_EPSILON);
}
inline double log_gamma_windschitl(double x) { return 0.918938533204673 + (x - 0.5) * std::log(x) - x + 0.5 * x * std::log(x * std::sinh(1 / x) + 1 / (810.0 * std::pow(x, 6.0))); }
inline double log_gamma_lanczos(double x)
{
    static const double q[7] = {75122.6331530, 80916.6278952, 36308.2951477, 8687.24529705, 1168.92649479, 83.8676043424, 2.50662827511};
    double a = (x + 0.5) * std::log(x + 5.5) - (x + 5.5);
    double b = 0;
    for (int n = 0; n < 7; ++n) {
        a -= std::log(x + double(n));
        b += q[n] * std::pow(x, double(n));
    }
    return a + std::log(b);
}
inline double log_gamma(double x) { return x > 15.0 ? log_gamma_windschitl(x) : log_gamma_lanczos(x); }

/* Optional statistics of one lsd_orc_detect call (lsd_orc_detect_stats), in the terms of the GPU seed loop (cs_lsd.cu: k_lsd_grow_seq keeps
 * the first LSD_SEQ_SCAP = 2 048 entries of a seed's region list in shared memory, the rest in HBM; the refine re-grow is written behind the
 * first pass, at base = first-pass size, so a seed's list holds n_all = first pass + re-grow entries, or the first pass alone when refine
 * did not re-grow).  Collecting them changes no result. */
enum {
    ST_SEEDS = 0,          /* seeds grown (region_grow from the raster scan) */
    ST_FIRST_SUM,          /* sum of first-pass region sizes */
    ST_NALL_SPILL,         /* seeds with n_all > 2 048 */
    ST_REGROW_PAST,        /* refine re-grows that start at list position >= 2 048 */
    ST_REDUCE_PAST,        /* reduce_region_radius iterations on a list (base + region) longer than 2 048 */
    ST_FIRST_MAX,          /* largest first pass */
    ST_NALL_MAX,           /* largest n_all */
    ST_FIRST_2047,         /* first passes of exactly 2 047, 2 048, 2 049 entries (three slots) */
    ST_NALL_2047 = ST_FIRST_2047 + 3, /* n_all of exactly 2 047, 2 048, 2 049 (three slots) */
    ST_NFA_MAX_N = ST_NALL_2047 + 3,  /* largest n of an nfa() call */
    ST_NFA_PAST_TABLE,     /* nfa() calls that evaluate log_gamma(k + 1) or log_gamma(n - k + 1) at an argument >= 16 384 */
    ST_COUNT
};
const int kSpill = 2048;         /* cs_lsd.cu LSD_SEQ_SCAP */
const int kLgammaTable = 16384;  /* cs_nfa.cuh CS_LGAMMA_TABLE */
thread_local int64_t *t_stats = nullptr;

/* lsd.cpp:1100-1136 (lsd_first_term) or descriptor.hpp:763-830 (log_gamma(n + 1) as the first term).  i_break: the i at which the tail
 * loop broke, n + 1 when it ran to the end, -1 for the early returns and the underflow branch. */
double nfa_tail(int n, int k, double p, double logNT, bool lsd_first_term, int *i_break)
{
    if (i_break) *i_break = -1;
    if (t_stats && n > t_stats[ST_NFA_MAX_N]) t_stats[ST_NFA_MAX_N] = n;
    if (n == 0 || k == 0) return -logNT;
    if (n == k) return -logNT - double(n) * std::log10(p);
    if (t_stats && (k + 1 >= kLgammaTable || n - k + 1 >= kLgammaTable)) t_stats[ST_NFA_PAST_TABLE]++;
    const double p_term = p / (1 - p);
    const double first = lsd_first_term ? (double(n) + 1) : log_gamma(double(n) + 1.0);
    const double log1term = first - log_gamma(double(k) + 1) - log_gamma(double(n - k) + 1) + double(k) * std::log(p) + double(n - k) * std::log(1.0 - p);
    double term = std::exp(log1term);
    if (double_equal(term, 0)) {
        if (k > n * p) return -log1term / kLN10 - logNT;
        return -logNT;
    }
    double bin_tail = term;
    const double tolerance = 0.1;
    int i = k + 1;
    for (; i <= n; ++i) {
        const double bin_term = double(n - i + 1) / double(i);
        const double mult_term = bin_term * p_term;
        term *= mult_term;
        bin_tail += term;
        if (bin_term < 1) {
            const double err = term * ((1 - std::pow(mult_term, double(n - i + 1))) / (1 - mult_term) - 1);
            if (err < tolerance * std::fabs(-std::log10(bin_tail) - logNT) * bin_tail) break;
        }
    }
    if (i_break) *i_break = i;
    return -std::log10(bin_tail) - logNT;
}

struct Rect {
    double x1, y1, x2, y2, width, x, y, theta, dx, dy, prec, p;
};

struct Lsd {
    int W = 0, H = 0;
    std::vector<double> img, angles, modgrad;
    std::vector<uint8_t> used;
    std::vector<int> list;  /* pixel addresses in pseudo-order (descending gradient bins) */
    std::vector<int> reg;   /* region: pixel addresses (angle / modgrad are looked up, they never change) */
    double LOG_NT = 0;
    int cur_base = 0, cur_n_all = 0; /* statistics: where the current seed's re-grow starts in the GPU's region list, and the list's length */

    /* lsd.cpp:1138-1154 */
    bool is_aligned(int address, double theta, double prec) const
    {
        if (address < 0) return false;
        const double a = angles[address];
        if (a == kNOTDEF) return false;
        double n_theta = theta - a;
        if (n_theta < 0) n_theta = -n_theta;
        if (n_theta > kM_3_2_PI) {
            n_theta -= kM_2__PI;
            if (n_theta < 0) n_theta = -n_theta;
        }
        return n_theta <= prec;
    }

    /* lsd.cpp:538-635 */
    void ll_angle(double threshold, unsigned n_bins)
    {
        angles.assign((size_t)W * H, 0.0);
        modgrad.assign((size_t)W * H, 0.0);
        for (int x = 0; x < W; x++) angles[(size_t)(H - 1) * W + x] = kNOTDEF;
        for (int y = 0; y < H; y++) angles[(size_t)y * W + W - 1] = kNOTDEF;
        double max_grad = -1;
        for (int y = 0; y < H - 1; ++y)
            for (int addr = y * W, addr_end = addr + W - 1; addr < addr_end; ++addr) {
                const double DA = img[addr + W + 1] - img[addr];
                const double BC = img[addr + 1] - img[addr + W];
                const double gx = DA + BC, gy = DA - BC;
                const double norm = std::sqrt((gx * gx + gy * gy) / 4);
                modgrad[addr] = norm;
                if (norm <= threshold)
                    angles[addr] = kNOTDEF;
                else {
                    angles[addr] = fast_atan2(float(gx), float(-gy)) * kDegToRads;
                    if (norm > max_grad) max_grad = norm;
                }
            }
        /* The order seeds are visited in.  ll_angle (lsd.cpp:588-634) files every pixel into one of 1024 gradient bins and links the bins,
         * highest first, through coorlist::next -- but the nodes live in a std::vector filled in RASTER order (count increments with the scan),
         * and flsd walks that vector by index (lsd.cpp:478-480: `for i < list.size(): adx = list[i].p.x + list[i].p.y * img_width`), never
         * through the links.  So the reference visits seeds in raster order over x < W - 1, y < H - 1; the pseudo-ordering is dead code in this
         * vendored file.  (Round 1 restated the links, not the loop: compiled from its own source -- oracle/ref/lsd_ref.cpp -- the reference
         * reproduces all 271 segments of its shipped 0000_edge.txt, the round-1 restatement reproduced 116.)  The vector has W * H nodes; the
         * ones past (W - 1)(H - 1) keep their default point (0, 0), a seed already used by then. */
        (void)n_bins;
        (void)max_grad;
        list.assign((size_t)(W - 1) * (H - 1), 0);
        size_t k = 0;
        for (int y = 0; y < H - 1; ++y)
            for (int x = 0; x < W - 1; ++x) list[k++] = y * W + x;
    }

    /* lsd.cpp:637-688 */
    void region_grow(int s_addr, int &reg_size, double &reg_angle, double prec)
    {
        reg_size = 1;
        reg[0] = s_addr;
        reg_angle = angles[s_addr];
        float sumdx = float(std::cos(reg_angle));
        float sumdy = float(std::sin(reg_angle));
        used[s_addr] = 1;
        for (int i = 0; i < reg_size; ++i) {
            const int px = reg[i] % W, py = reg[i] / W;
            const int xx_min = std::max(px - 1, 0), xx_max = std::min(px + 1, W - 1);
            const int yy_min = std::max(py - 1, 0), yy_max = std::min(py + 1, H - 1);
            for (int yy = yy_min; yy <= yy_max; ++yy) {
                int c_addr = xx_min + yy * W;
                for (int xx = xx_min; xx <= xx_max; ++xx, ++c_addr) {
                    if ((used[c_addr] != 1) && is_aligned(c_addr, reg_angle, prec)) {
                        used[c_addr] = 1;
                        reg[reg_size] = c_addr;
                        ++reg_size;
                        const double angle = angles[c_addr];
                        /* the reference's cos(float(angle)) is libm's cosf, whose last bit varies between libm versions; the
                         * build pins it to the correctly rounded value, computed through double on both the oracle and the GPU */
                        sumdx += (float)std::cos((double)float(angle));
                        sumdy += (float)std::sin((double)float(angle));
                        reg_angle = fast_atan2(sumdy, sumdx) * kDegToRads;
                    }
                }
            }
        }
    }

    /* lsd.cpp:748-784 */
    double get_theta(int reg_size, double x, double y, double reg_angle, double prec) const
    {
        double Ixx = 0.0, Iyy = 0.0, Ixy = 0.0;
        for (int i = 0; i < reg_size; ++i) {
            const double regx = reg[i] % W, regy = reg[i] / W;
            const double weight = modgrad[reg[i]];
            const double dx = regx - x, dy = regy - y;
            Ixx += dy * dy * weight;
            Iyy += dx * dx * weight;
            Ixy -= dx * dy * weight;
        }
        const double lambda = 0.5 * (Ixx + Iyy - std::sqrt((Ixx - Iyy) * (Ixx - Iyy) + 4.0 * Ixy * Ixy));
        double theta = (std::fabs(Ixx) > std::fabs(Iyy)) ? double(fast_atan2(float(lambda - Ixx), float(Ixy))) : double(fast_atan2(float(Ixy), float(lambda - Iyy)));
        theta *= kDegToRads;
        if (angle_diff(theta, reg_angle) > prec) theta += kPI;
        return theta;
    }

    /* lsd.cpp:690-746 */
    void region2rect(int reg_size, double reg_angle, double prec, double p, Rect &rec) const
    {
        double x = 0, y = 0, sum = 0;
        for (int i = 0; i < reg_size; ++i) {
            const double weight = modgrad[reg[i]];
            x += double(reg[i] % W) * weight;
            y += double(reg[i] / W) * weight;
            sum += weight;
        }
        x /= sum;
        y /= sum;
        const double theta = get_theta(reg_size, x, y, reg_angle, prec);
        const double dx = std::cos(theta), dy = std::sin(theta);
        double l_min = 0, l_max = 0, w_min = 0, w_max = 0;
        for (int i = 0; i < reg_size; ++i) {
            const double regdx = double(reg[i] % W) - x, regdy = double(reg[i] / W) - y;
            const double l = regdx * dx + regdy * dy;
            const double w = -regdx * dy + regdy * dx;
            if (l > l_max)
                l_max = l;
            else if (l < l_min)
                l_min = l;
            if (w > w_max)
                w_max = w;
            else if (w < w_min)
                w_min = w;
        }
        rec.x1 = x + l_min * dx;
        rec.y1 = y + l_min * dy;
        rec.x2 = x + l_max * dx;
        rec.y2 = y + l_max * dy;
        rec.width = w_max - w_min;
        rec.x = x;
        rec.y = y;
        rec.theta = theta;
        rec.dx = dx;
        rec.dy = dy;
        rec.prec = prec;
        rec.p = p;
        if (rec.width < 1.0) rec.width = 1.0;
    }

    /* lsd.cpp:834-871 */
    bool reduce_region_radius(int &reg_size, double reg_angle, double prec, double p, Rect &rec, double density, double density_th)
    {
        const double xc = double(reg[0] % W), yc = double(reg[0] / W);
        const double radSq1 = dist_sq(xc, yc, rec.x1, rec.y1), radSq2 = dist_sq(xc, yc, rec.x2, rec.y2);
        double radSq = radSq1 > radSq2 ? radSq1 : radSq2;
        while (density < density_th) {
            if (t_stats && cur_base + reg_size > kSpill) t_stats[ST_REDUCE_PAST]++;
            radSq *= 0.75 * 0.75;
            for (int i = 0; i < reg_size; ++i) {
                if (dist_sq(xc, yc, double(reg[i] % W), double(reg[i] / W)) > radSq) {
                    used[reg[i]] = 0;
                    std::swap(reg[i], reg[reg_size - 1]);
                    --reg_size;
                    --i;
                }
            }
            if (reg_size < 2) return false;
            region2rect(reg_size, reg_angle, prec, p, rec);
            density = double(reg_size) / (dist2(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
        }
        return true;
    }

    /* lsd.cpp:786-832 */
    bool refine(int &reg_size, double reg_angle, double prec, double p, Rect &rec, double density_th)
    {
        double density = double(reg_size) / (dist2(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
        if (density >= density_th) return true;
        const double xc = double(reg[0] % W), yc = double(reg[0] / W);
        const double ang_c = angles[reg[0]];
        double sum = 0, s_sum = 0;
        int n = 0;
        for (int i = 0; i < reg_size; ++i) {
            used[reg[i]] = 0;
            if (dist2(xc, yc, reg[i] % W, reg[i] / W) < rec.width) {
                const double ang_d = angle_diff_signed(angles[reg[i]], ang_c);
                sum += ang_d;
                s_sum += ang_d * ang_d;
                ++n;
            }
        }
        const double mean_angle = sum / double(n);
        const double tau = 2.0 * std::sqrt((s_sum - 2.0 * mean_angle * sum) / double(n) + mean_angle * mean_angle);
        cur_base = reg_size;
        if (t_stats && cur_base >= kSpill) t_stats[ST_REGROW_PAST]++;
        region_grow(reg[0], reg_size, reg_angle, tau);
        cur_n_all = cur_base + reg_size;
        if (reg_size < 2) return false;
        region2rect(reg_size, reg_angle, prec, p, rec);
        density = double(reg_size) / (dist2(rec.x1, rec.y1, rec.x2, rec.y2) * rec.width);
        if (density < density_th) return reduce_region_radius(reg_size, reg_angle, prec, p, rec, density, density_th);
        return true;
    }

    /* lsd.cpp:1100-1136 */
    double nfa(int n, int k, double p) const { return nfa_tail(n, k, p, LOG_NT, true, nullptr); }

    /* lsd.cpp:977-1098, including the vendored slips (tailp->p.x where y is meant; int/int slopes) */
    double rect_nfa(const Rect &rec) const
    {
        int total_pts = 0, alg_pts = 0;
        const double half_width = rec.width / 2.0;
        const double dyhw = rec.dy * half_width, dxhw = rec.dx * half_width;
        struct E {
            int x, y;
            bool taken;
        } o[4];
        o[0] = {int(rec.x1 - dyhw), int(rec.y1 + dxhw), false};
        o[1] = {int(rec.x2 - dyhw), int(rec.y2 + dxhw), false};
        o[2] = {int(rec.x2 + dyhw), int(rec.y2 - dxhw), false};
        o[3] = {int(rec.x1 + dyhw), int(rec.y1 - dxhw), false};
        /* std::sort of 4 elements by (x, then y): insertion sort yields the same order (the comparator is a strict weak order
         * and equal keys are indistinguishable) */
        for (int i = 1; i < 4; i++) {
            E v = o[i];
            int j = i - 1;
            while (j >= 0 && ((v.x == o[j].x) ? (v.y < o[j].y) : (v.x < o[j].x))) {
                o[j + 1] = o[j];
                j--;
            }
            o[j + 1] = v;
        }
        E *min_y = &o[0], *max_y = &o[0];
        for (unsigned i = 1; i < 4; ++i) {
            if (min_y->y > o[i].y) min_y = &o[i];
            if (max_y->y < o[i].y) max_y = &o[i];
        }
        min_y->taken = true;
        E *leftmost = 0;
        for (unsigned i = 0; i < 4; ++i)
            if (!o[i].taken) {
                if (!leftmost)
                    leftmost = &o[i];
                else if (leftmost->x > o[i].x)
                    leftmost = &o[i];
            }
        leftmost->taken = true;
        E *rightmost = 0;
        for (unsigned i = 0; i < 4; ++i)
            if (!o[i].taken) {
                if (!rightmost)
                    rightmost = &o[i];
                else if (rightmost->x < o[i].x)
                    rightmost = &o[i];
            }
        rightmost->taken = true;
        E *tailp = 0;
        for (unsigned i = 0; i < 4; ++i)
            if (!o[i].taken) {
                if (!tailp)
                    tailp = &o[i];
                else if (tailp->x > o[i].x)
                    tailp = &o[i];
            }
        tailp->taken = true;
        const double flstep = (min_y->y != leftmost->y) ? (min_y->x - leftmost->x) / (min_y->y - leftmost->y) : 0;
        const double slstep = (leftmost->y != tailp->x) ? (leftmost->x - tailp->x) / (leftmost->y - tailp->x) : 0;
        const double frstep = (min_y->y != rightmost->y) ? (min_y->x - rightmost->x) / (min_y->y - rightmost->y) : 0;
        const double srstep = (rightmost->y != tailp->x) ? (rightmost->x - tailp->x) / (rightmost->y - tailp->x) : 0;
        double lstep = flstep, rstep = frstep;
        double left_x = min_y->x, right_x = min_y->x;
        const int min_iter = min_y->y, max_iter = max_y->y;
        for (int y = min_iter; y <= max_iter; ++y) {
            if (y < 0 || y >= H) continue;
            int adx = y * W + int(left_x);
            for (int x = int(left_x); x <= int(right_x); ++x, ++adx) {
                if (x < 0 || x >= W) continue;
                ++total_pts;
                if (is_aligned(adx, rec.theta, rec.prec)) ++alg_pts;
            }
            if (y >= leftmost->y) lstep = slstep;
            if (y >= rightmost->y) rstep = srstep;
            left_x += lstep;
            right_x += rstep;
        }
        return nfa(total_pts, alg_pts, rec.p);
    }

    /* lsd.cpp:873-975 */
    double rect_improve(Rect &rec) const
    {
        const double delta = 0.5, delta_2 = delta / 2.0, LOG_EPS = 0;
        double log_nfa = rect_nfa(rec);
        if (log_nfa > LOG_EPS) return log_nfa;
        Rect r = rec;
        for (int n = 0; n < 5; ++n) {
            r.p /= 2;
            r.prec = r.p * kPI;
            const double v = rect_nfa(r);
            if (v > log_nfa) {
                log_nfa = v;
                rec = r;
            }
        }
        if (log_nfa > LOG_EPS) return log_nfa;
        r = rec;
        for (unsigned n = 0; n < 5; ++n)
            if ((r.width - delta) >= 0.5) {
                r.width -= delta;
                const double v = rect_nfa(r);
                if (v > log_nfa) {
                    rec = r;
                    log_nfa = v;
                }
            }
        if (log_nfa > LOG_EPS) return log_nfa;
        r = rec;
        for (unsigned n = 0; n < 5; ++n)
            if ((r.width - delta) >= 0.5) {
                r.x1 += -r.dy * delta_2;
                r.y1 += r.dx * delta_2;
                r.x2 += -r.dy * delta_2;
                r.y2 += r.dx * delta_2;
                r.width -= delta;
                const double v = rect_nfa(r);
                if (v > log_nfa) {
                    rec = r;
                    log_nfa = v;
                }
            }
        if (log_nfa > LOG_EPS) return log_nfa;
        r = rec;
        for (unsigned n = 0; n < 5; ++n)
            if ((r.width - delta) >= 0.5) {
                r.x1 -= -r.dy * delta_2;
                r.y1 -= r.dx * delta_2;
                r.x2 -= -r.dy * delta_2;
                r.y2 -= r.dx * delta_2;
                r.width -= delta;
                const double v = rect_nfa(r);
                if (v > log_nfa) {
                    rec = r;
                    log_nfa = v;
                }
            }
        if (log_nfa > LOG_EPS) return log_nfa;
        r = rec;
        for (unsigned n = 0; n < 5; ++n)
            if ((r.width - delta) >= 0.5) {
                r.p /= 2;
                r.prec = r.p * kPI;
                const double v = rect_nfa(r);
                if (v > log_nfa) {
                    rec = r;
                    log_nfa = v;
                }
            }
        return log_nfa;
    }
};

}  // namespace

extern "C" float lsd_orc_fast_atan2(float y, float x) { return fast_atan2(y, x); }

/* the two OpenCV primitives of lsd.cpp:457-459 on their own (oracle/ref/minicv.hpp forwards cv::GaussianBlur / cv::resize to them when the
 * reference's lsd.cpp is compiled into oracle/_ref) */
extern "C" void lsd_orc_gaussian7(const double *src, int w, int h, double *dst)
{
    std::vector<double> s(src, src + (size_t)w * h), b;
    gaussian_blur7(s, w, h, b);
    std::memcpy(dst, b.data(), sizeof(double) * b.size());
}
extern "C" void lsd_orc_resize(const double *src, int w, int h, double scale, double *dst, int *dw, int *dh)
{
    std::vector<double> s(src, src + (size_t)w * h), r;
    int W = 0, H = 0;
    resize_linear(s, w, h, scale, r, W, H);
    std::memcpy(dst, r.data(), sizeof(double) * r.size());
    *dw = W;
    *dh = H;
}

extern "C" void lsd_orc_blur_resize(const double *src, int w, int h, double *blur_out, double *scaled_out, int *dw, int *dh)
{
    std::vector<double> s(src, src + (size_t)w * h), b, r;
    gaussian_blur7(s, w, h, b);
    if (blur_out) std::memcpy(blur_out, b.data(), sizeof(double) * b.size());
    int ow, oh;
    resize_linear(b, w, h, 0.8, r, ow, oh);
    if (scaled_out) std::memcpy(scaled_out, r.data(), sizeof(double) * r.size());
    *dw = ow;
    *dh = oh;
}

/* line_lbd_detect::detect_filter_lines with use_LSD = true, one octave (line_lbd_allclass.cpp:216-221).
 * raw_lines (optional): every LSD segment before the KeyLine filters, cap_raw x 4; stage buffers optional. */
extern "C" int lsd_orc_detect(const uint8_t *img, int w, int h, int stride, int channels, float line_length_thres, float *lines_out, int cap,
                              float *raw_lines, int cap_raw, int *n_raw_out, double *scaled_out, double *modgrad_out, double *angles_out,
                              int32_t *list_out, int *list_len, int refine_mode /* 2 = LSD_REFINE_ADV (the reference), 1 = STD, 0 = NONE (pinning only) */)
{
    /* LSDDetector::detectImpl :156-160 */
    std::vector<uint8_t> gray((size_t)w * h);
    if (channels != 1)
        orc_bgr2gray(img, w, h, stride, gray.data(), w, 1);
    else
        for (int y = 0; y < h; y++) std::memcpy(&gray[(size_t)y * w], img + (size_t)y * stride, w);
    std::vector<double> image((size_t)w * h);
    for (size_t i = 0; i < image.size(); i++) image[i] = gray[i];

    /* flsd :440-536 with the default parameters */
    const double SCALE = 0.8, ANG_TH = 22.5, QUANT = 2.0, LOG_EPS = 0, DENSITY_TH = 0.7;
    const double prec = kPI * ANG_TH / 180, p = ANG_TH / 180, rho = QUANT / std::sin(prec);
    Lsd L;
    {
        std::vector<double> blurred;
        gaussian_blur7(image, w, h, blurred); /* sigma = 0.6/0.8, ksize = 1 + 2*ceil(sigma*sqrt(2*3*ln 10)) = 7 */
        resize_linear(blurred, w, h, SCALE, L.img, L.W, L.H);
    }
    L.ll_angle(rho, 1024);
    L.LOG_NT = 5 * (std::log10(double(L.W)) + std::log10(double(L.H))) / 2 + std::log10(11.0);
    const int min_reg_size = int(-L.LOG_NT / std::log10(p));
    L.used.assign((size_t)L.W * L.H, 0);
    L.reg.assign((size_t)L.W * L.H, 0);
    if (scaled_out) std::memcpy(scaled_out, L.img.data(), sizeof(double) * L.img.size());
    if (modgrad_out) std::memcpy(modgrad_out, L.modgrad.data(), sizeof(double) * L.modgrad.size());
    if (angles_out) std::memcpy(angles_out, L.angles.data(), sizeof(double) * L.angles.size());
    if (list_out && list_len) {
        std::memcpy(list_out, L.list.data(), sizeof(int32_t) * L.list.size());
        *list_len = (int)L.list.size();
    }

    std::vector<float> lines; /* Vec4f */
    for (size_t i = 0; i < L.list.size(); ++i) {
        const int adx = L.list[i];
        if (L.used[adx] == 0 && L.angles[adx] != kNOTDEF) {
            int reg_size;
            double reg_angle;
            L.region_grow(adx, reg_size, reg_angle, prec);
            L.cur_base = 0;
            L.cur_n_all = reg_size;
            if (t_stats) {
                t_stats[ST_SEEDS]++;
                t_stats[ST_FIRST_SUM] += reg_size;
                t_stats[ST_FIRST_MAX] = std::max<int64_t>(t_stats[ST_FIRST_MAX], reg_size);
                if (std::abs(reg_size - kSpill) <= 1) t_stats[ST_FIRST_2047 + reg_size - (kSpill - 1)]++;
            }
            /* the seed's list length once region_grow / refine are done with it */
            auto note_n_all = [&L]() {
                if (!t_stats) return;
                const int n_all = L.cur_n_all;
                if (n_all > kSpill) t_stats[ST_NALL_SPILL]++;
                t_stats[ST_NALL_MAX] = std::max<int64_t>(t_stats[ST_NALL_MAX], n_all);
                if (std::abs(n_all - kSpill) <= 1) t_stats[ST_NALL_2047 + n_all - (kSpill - 1)]++;
            };
            if (reg_size < min_reg_size) {
                note_n_all();
                continue;
            }
            Rect rec;
            L.region2rect(reg_size, reg_angle, prec, p, rec);
            const bool refined = refine_mode > 0 && L.refine(reg_size, reg_angle, prec, p, rec, DENSITY_TH);
            note_n_all();
            if (refine_mode > 0) {
                if (!refined) continue;
                if (refine_mode >= 2) {
                    const double log_nfa = L.rect_improve(rec);
                    if (log_nfa <= LOG_EPS) continue;
                }
            }
            rec.x1 += 0.5;
            rec.y1 += 0.5;
            rec.x2 += 0.5;
            rec.y2 += 0.5;
            rec.x1 /= SCALE;
            rec.y1 /= SCALE;
            rec.x2 /= SCALE;
            rec.y2 /= SCALE;
            lines.push_back(float(rec.x1));
            lines.push_back(float(rec.y1));
            lines.push_back(float(rec.x2));
            lines.push_back(float(rec.y2));
        }
    }
    const int n_raw = (int)lines.size() / 4;
    if (n_raw_out) *n_raw_out = n_raw;
    if (raw_lines) std::memcpy(raw_lines, lines.data(), sizeof(float) * 4 * std::min(n_raw, cap_raw));

    /* LSDDetector::detectImpl :205-256 + filter_lines + keylines_to_mat */
    int n_out = 0;
    const float pre_boundary_thre = 10;
    for (int k = 0; k < n_raw; k++) {
        float e[4] = {lines[4 * k], lines[4 * k + 1], lines[4 * k + 2], lines[4 * k + 3]};
        /* checkLineExtremes :75-101 (octave image size == image size for one octave) */
        if (e[0] < 0) e[0] = 0;
        if (e[0] >= w) e[0] = (float)w - 1.0f;
        if (e[2] < 0) e[2] = 0;
        if (e[2] >= w) e[2] = (float)w - 1.0f;
        if (e[1] < 0) e[1] = 0;
        if (e[1] >= h) e[1] = (float)h - 1.0f;
        if (e[3] < 0) e[3] = 0;
        if (e[3] >= h) e[3] = (float)h - 1.0f;
        const float sx = e[0] * 1.0f, sy = e[1] * 1.0f, ex = e[2] * 1.0f, ey = e[3] * 1.0f; /* octaveScale = pow(scale, 0) */
        if (((sx < pre_boundary_thre) && (ex < pre_boundary_thre)) || ((sx > w - pre_boundary_thre) && (ex > w - pre_boundary_thre)) ||
            ((sy < pre_boundary_thre) && (ey < pre_boundary_thre)) || ((sy > h - pre_boundary_thre) && (ey > h - pre_boundary_thre)))
            continue;
        const float line_length = (float)std::sqrt(std::pow((double)(e[0] - e[2]), 2) + std::pow((double)(e[1] - e[3]), 2));
        if (!(line_length > line_length_thres)) continue; /* filter_lines: octave == 0 && lineLength > thres */
        if (n_out < cap) {
            lines_out[4 * n_out + 0] = sx;
            lines_out[4 * n_out + 1] = sy;
            lines_out[4 * n_out + 2] = ex;
            lines_out[4 * n_out + 3] = ey;
        }
        n_out++;
    }
    return n_out;
}

/* lsd_orc_detect with its statistics (stats: ST_COUNT = 15 int64, zeroed here; see the enum above) */
extern "C" int lsd_orc_detect_stats(const uint8_t *img, int w, int h, int stride, int channels, float line_length_thres, float *lines_out, int cap,
                                    float *raw_lines, int cap_raw, int *n_raw_out, int refine_mode, int64_t *stats)
{
    static_assert(ST_COUNT == 15, "pyoracle.LSD_STAT_NAMES names 15 slots");
    std::memset(stats, 0, sizeof(int64_t) * ST_COUNT);
    t_stats = stats;
    const int n = lsd_orc_detect(img, w, h, stride, channels, line_length_thres, lines_out, cap, raw_lines, cap_raw, n_raw_out, nullptr, nullptr,
                                 nullptr, nullptr, nullptr, refine_mode);
    t_stats = nullptr;
    return n;
}

/* the reference's nfa on its own: lsd.cpp's ((n + 1) first term, lsd_first_term = 1) or descriptor.hpp's (log_gamma(n + 1)); i_break: the i at
 * which the tail loop stopped (n + 1: it ran to the end), -1 for the early returns and the underflow branch */
extern "C" double orc_lsd_nfa(int n, int k, double p, double logNT, int lsd_first_term, int *i_break)
{
    return nfa_tail(n, k, p, logNT, lsd_first_term != 0, i_break);
}

/* the same over arrays (one logNT and form for all) */
extern "C" void orc_lsd_nfa_many(const int32_t *n, const int32_t *k, const double *p, int count, double logNT, int lsd_first_term, double *out,
                                 int32_t *i_break)
{
    for (int i = 0; i < count; i++) {
        int b = -1;
        out[i] = nfa_tail(n[i], k[i], p[i], logNT, lsd_first_term != 0, &b);
        i_break[i] = b;
    }
}
