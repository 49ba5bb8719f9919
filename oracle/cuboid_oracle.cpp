/*
 * oracle/cuboid_oracle.cpp -- CPU ORACLE for the cuboid proposal path.  TEST INFRASTRUCTURE ONLY.
 *
 * A dependency-free (no Eigen / OpenCV / ROS) restatement of
 *   detect_3d_cuboid/src/box_proposal_detail.cpp:36-557   (set_cam_pose, detect_cuboid)
 *   detect_3d_cuboid/src/object_3d_util.cpp:141-648        (geometry + scoring primitives)
 *   detect_3d_cuboid/src/matrix_utils.cpp:36-46,75-89,159-176,316-335,350-363
 * plus the three OpenCV calls on the path (cvtColor / Canny / distanceTransform), restated
 * from OpenCV's published algorithms and pinned bit-for-bit to the in-container cv2 4.13.
 *
 * PARITY: PINNED to the reference.  It ships no tests or expected C++ outputs, but its own sources (matrix_utils.cpp, object_3d_util.cpp,
 * box_proposal_detail.cpp) compile from /root/reference against oracle/ref/minieigen.hpp / minicv.hpp into oracle/_ref/libcuboid_ref.so,
 * and every field of every cuboid that library returns equals this restatement's, == on doubles, in every mode tried (default, top-k,
 * roll / pitch sampling with several boxes, no height samples, one configuration; tests/test_oracle_ref_detect_cuboid.py; with libm's
 * atan2 on both sides -- the parity tests against CUDA use the arithmetic atan2 of pmath.h, tied to libm by tests/test_pmath.py).
 * The OpenCV stages are bit-exact against cv2; and, run on the shipped object_slam sequence at the shipped per-frame poses, this oracle
 * lands on the cuboids the authors ship from their MATLAB implementation (object_slam/data/detect_cuboids_saved.txt) up to the sampling
 * grid -- median 3.2 cm, same yaw sample on most frames (tests/test_oracle_matlab_crosscheck.py), a soft cross-check.
 * Build with -O2 -ffp-contract=off (no FMA contraction) so + - * / sqrt are IEEE-exact and comparable with the CUDA path compiled with
 * -fmad=false.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) use this.
 */
#include "orc_api.h"
#include "pmath.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <numeric>
#include <vector>

/* atan2 of the angle-error chain (merge_break_lines, VP_support_edge_infos, box_edge_alignment_angle_error; object_3d_util.cpp:167-172,
 * 321,392,480).  1 (default): the arithmetic definition shared with the CUDA path (pmath.h), so that parity is bit for bit;
 * 0: libm's, what the reference itself calls -- the two differ by at most one ulp (tests/test_pmath.py), which matters only where
 * fuse_normalize_scores_v2 splits a pair of mathematically equal angle errors (see orc_last_cut_margin below). */
static thread_local int g_portable_atan2 = 1;
extern "C" void orc_set_portable_atan2(int on) { g_portable_atan2 = on; }
extern "C" double orc_atan2_portable(double y, double x) { return orc_pm_atan2(y, x); }
static inline double ang_atan2(double y, double x) { return g_portable_atan2 ? orc_pm_atan2(y, x) : std::atan2(y, x); }

namespace {

struct P2 {
    double x, y;
};

inline P2 sub(P2 a, P2 b) { return {a.x - b.x, a.y - b.y}; }
inline double norm2(P2 a) { return std::sqrt(a.x * a.x + a.y * a.y); }

/* ------------------------------------------------------------------ small dense algebra */
/* 3x3 inverse by cofactors in the evaluation order Eigen uses for fixed 3x3 (Inverse_3x3 helper):
 * first-column cofactors, determinant from them, then every cofactor times 1/det. */
inline double cof3(const double *m, int i, int j)
{
    const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
    return m[i1 * 3 + j1] * m[i2 * 3 + j2] - m[i1 * 3 + j2] * m[i2 * 3 + j1];
}
void inv3(const double *m, double *r)
{
    const double c00 = cof3(m, 0, 0), c10 = cof3(m, 1, 0), c20 = cof3(m, 2, 0);
    const double det = (c00 * m[0] + c10 * m[3]) + c20 * m[6];
    const double invdet = 1.0 / det;
    r[0] = c00 * invdet;
    r[1] = c10 * invdet;
    r[2] = c20 * invdet;
    r[3] = cof3(m, 0, 1) * invdet;
    r[4] = cof3(m, 1, 1) * invdet;
    r[5] = cof3(m, 2, 1) * invdet;
    r[6] = cof3(m, 0, 2) * invdet;
    r[7] = cof3(m, 1, 2) * invdet;
    r[8] = cof3(m, 2, 2) * invdet;
}
void mul33(const double *a, const double *b, double *c)
{
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++)
            c[i * 3 + j] = (a[i * 3 + 0] * b[0 * 3 + j] + a[i * 3 + 1] * b[1 * 3 + j]) + a[i * 3 + 2] * b[2 * 3 + j];
}

/* matrix_utils.cpp:75-89 euler_zyx_to_rot */
void euler_zyx_to_rot(double roll, double pitch, double yaw, double *R)
{
    const double cp = std::cos(pitch), sp = std::sin(pitch);
    const double sr = std::sin(roll), cr = std::cos(roll);
    const double sy = std::sin(yaw), cy = std::cos(yaw);
    R[0] = cp * cy;
    R[1] = (sr * sp * cy) - (cr * sy);
    R[2] = (cr * sp * cy) + (sr * sy);
    R[3] = cp * sy;
    R[4] = (sr * sp * sy) + (cr * cy);
    R[5] = (cr * sp * sy) - (sr * cy);
    R[6] = -sp;
    R[7] = sr * cp;
    R[8] = cr * cp;
}

/* Eigen::Quaterniond(Matrix3d) (Shepperd branches), then matrix_utils.cpp:36-46 quat_to_euler_zyx */
void rot_to_euler_via_quat(const double *m, double *euler)
{
    double q[4]; /* x y z w */
    double t = m[0] + m[4] + m[8];
    if (t > 0.0) {
        t = std::sqrt(t + 1.0);
        q[3] = 0.5 * t;
        t = 0.5 / t;
        q[0] = (m[2 * 3 + 1] - m[1 * 3 + 2]) * t;
        q[1] = (m[0 * 3 + 2] - m[2 * 3 + 0]) * t;
        q[2] = (m[1 * 3 + 0] - m[0 * 3 + 1]) * t;
    } else {
        int i = 0;
        if (m[4] > m[0]) i = 1;
        if (m[8] > m[i * 3 + i]) i = 2;
        const int j = (i + 1) % 3, k = (j + 1) % 3;
        t = std::sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0);
        q[i] = 0.5 * t;
        t = 0.5 / t;
        q[3] = (m[k * 3 + j] - m[j * 3 + k]) * t;
        q[j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
        q[k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
    }
    const double qx = q[0], qy = q[1], qz = q[2], qw = q[3];
    euler[0] = std::atan2(2 * (qw * qx + qy * qz), 1 - 2 * (qx * qx + qy * qy));
    euler[1] = std::asin(2 * (qw * qy - qz * qx));
    euler[2] = std::atan2(2 * (qw * qz + qx * qy), 1 - 2 * (qy * qy + qz * qz));
}

/* struct cam_pose_infos (detect_3d_cuboid.h:39-51); projectionMatrix omitted: it is passed to
 * change_2d_corner_to_3d_object but never read there (object_3d_util.cpp:610-648). */
struct CamPose {
    double T[16];
    double K[9];
    double R[9];
    double euler[3];
    double invR[9];
    double invK[9];
    double KinvR[9];
    double yaw;
};

/* box_proposal_detail.cpp:42-54 */
void set_cam_pose(CamPose &cp, const double *T)
{
    std::memcpy(cp.T, T, sizeof(cp.T));
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) cp.R[i * 3 + j] = T[i * 4 + j];
    rot_to_euler_via_quat(cp.R, cp.euler);
    inv3(cp.R, cp.invR);
    mul33(cp.K, cp.invR, cp.KinvR);
    cp.yaw = cp.euler[2];
}

/* cam_pose.transToWolrd.transpose() * plane (box_proposal_detail.cpp:100,238,486) */
void plane_to_sensor(const double *T, const double *plane_world, double *plane_sensor)
{
    for (int i = 0; i < 4; i++)
        plane_sensor[i] = ((T[0 * 4 + i] * plane_world[0] + T[1 * 4 + i] * plane_world[1]) + T[2 * 4 + i] * plane_world[2]) +
                          T[3 * 4 + i] * plane_world[3];
}

/* matrix_utils.cpp:350-363 */
template <class T>
void linespace(T starting, T ending, T step, std::vector<T> &res)
{
    while (starting <= ending) {
        res.push_back(starting);
        starting += step;
        if (res.size() > 1000) break;
    }
}

/* matrix_utils.cpp:327-335 */
inline double normalize_to_pi(double angle)
{
    if (angle > M_PI / 2)
        return angle - M_PI;
    else if (angle < -M_PI / 2)
        return angle + M_PI;
    return angle;
}

/* object_3d_util.cpp:141-144 */
inline bool inside_box(P2 pt, P2 lt, P2 rb) { return lt.x <= pt.x && pt.x <= rb.x && lt.y <= pt.y && pt.y <= rb.y; }

/* object_3d_util.cpp:194-230 */
P2 seg_hit_boundary(P2 pt_start, P2 pt_end, double bx0, double by0, double bx1, double by1)
{
    const P2 direc = sub(pt_end, pt_start);
    P2 hit = {-1, -1};
    if (by0 == by1) {
        const double lambd = (by0 - pt_start.y) / direc.y;
        if (lambd >= 0) {
            const P2 tmp = {pt_start.x + lambd * direc.x, pt_start.y + lambd * direc.y};
            if (bx0 <= tmp.x && tmp.x <= bx1) {
                hit = tmp;
                hit.y = by0;
            }
        }
    }
    if (bx0 == bx1) {
        const double lambd = (bx0 - pt_start.x) / direc.x;
        if (lambd >= 0) {
            const P2 tmp = {pt_start.x + lambd * direc.x, pt_start.y + lambd * direc.y};
            if (by0 <= tmp.y && tmp.y <= by1) {
                hit = tmp;
                hit.x = bx0;
            }
        }
    }
    return hit;
}

/* object_3d_util.cpp:233-252, infinite_line = true */
P2 line_intersect(P2 p1s, P2 p1e, P2 p2s, P2 p2e)
{
    const double X2_X1 = p1e.x - p1s.x, Y2_Y1 = p1e.y - p1s.y;
    const double X4_X3 = p2e.x - p2s.x, Y4_Y3 = p2e.y - p2s.y;
    const double X1_X3 = p1s.x - p2s.x, Y1_Y3 = p1s.y - p2s.y;
    const double u_a = (X4_X3 * Y1_Y3 - Y4_Y3 * X1_X3) / (Y4_Y3 * X2_X1 - X4_X3 * Y2_Y1);
    return {p1s.x + X2_X1 * u_a, p1s.y + Y2_Y1 * u_a};
}

/* object_3d_util.cpp:602-607 (+ matrix_utils.cpp:159-168) */
void vanishing_points(const double *KinvR, double yaw, P2 &vp1, P2 &vp2, P2 &vp3)
{
    const double c = std::cos(yaw), s = std::sin(yaw);
    double h[3];
    for (int i = 0; i < 3; i++) h[i] = (KinvR[i * 3 + 0] * c + KinvR[i * 3 + 1] * s) + KinvR[i * 3 + 2] * 0.0;
    vp1 = {h[0] / h[2], h[1] / h[2]};
    for (int i = 0; i < 3; i++) h[i] = (KinvR[i * 3 + 0] * (-s) + KinvR[i * 3 + 1] * c) + KinvR[i * 3 + 2] * 0.0;
    vp2 = {h[0] / h[2], h[1] / h[2]};
    for (int i = 0; i < 3; i++) h[i] = (KinvR[i * 3 + 0] * 0.0 + KinvR[i * 3 + 1] * 0.0) + KinvR[i * 3 + 2] * 1.0;
    vp3 = {h[0] / h[2], h[1] / h[2]};
}

/* object_3d_util.cpp:300-376 */
int merge_break_lines(std::vector<double> &L, int n, double dist_thre, double angle_thre_deg, double len_thre)
{
    bool can_force_merge = true;
    int total = n, counter = 0;
    const double angle_thre = angle_thre_deg / 180.0 * M_PI;
    std::vector<double> ang(n > 0 ? n : 1);
    while (can_force_merge && counter < 500) {
        counter++;
        can_force_merge = false;
        for (int i = 0; i < total; i++) ang[i] = ang_atan2(L[i * 4 + 3] - L[i * 4 + 1], L[i * 4 + 2] - L[i * 4 + 0]);
        for (int s1 = 0; s1 < total - 1; s1++) {
            for (int s2 = s1 + 1; s2 < total; s2++) {
                const double diff = std::abs(ang[s1] - ang[s2]);
                const double angle_diff = std::min(diff, M_PI - diff);
                if (angle_diff < angle_thre) {
                    const double d12 = norm2({L[s1 * 4 + 2] - L[s2 * 4 + 0], L[s1 * 4 + 3] - L[s2 * 4 + 1]});
                    const double d21 = norm2({L[s2 * 4 + 2] - L[s1 * 4 + 0], L[s2 * 4 + 3] - L[s1 * 4 + 1]});
                    if (d12 < dist_thre || d21 < dist_thre) {
                        P2 ms, me;
                        if (L[s1 * 4 + 0] < L[s2 * 4 + 0])
                            ms = {L[s1 * 4 + 0], L[s1 * 4 + 1]};
                        else
                            ms = {L[s2 * 4 + 0], L[s2 * 4 + 1]};
                        if (L[s1 * 4 + 2] > L[s2 * 4 + 2])
                            me = {L[s1 * 4 + 2], L[s1 * 4 + 3]};
                        else
                            me = {L[s2 * 4 + 2], L[s2 * 4 + 3]};
                        const double merged_angle = ang_atan2(me.y - ms.y, me.x - ms.x);
                        const double temp = std::abs(ang[s1] - merged_angle);
                        const double merge_angle_diff = std::min(temp, M_PI - temp);
                        if (merge_angle_diff < angle_thre) {
                            L[s1 * 4 + 0] = ms.x;
                            L[s1 * 4 + 1] = ms.y;
                            L[s1 * 4 + 2] = me.x;
                            L[s1 * 4 + 3] = me.y;
                            /* fast_RemoveRow (matrix_utils.cpp:172-176) */
                            for (int c = 0; c < 4; c++) L[s2 * 4 + c] = L[(total - 1) * 4 + c];
                            total--;
                            can_force_merge = true;
                            break;
                        }
                    }
                }
            }
            if (can_force_merge) break;
        }
    }
    if (len_thre > 0) {
        int keep = 0;
        for (int i = 0; i < total; i++) {
            const double len = norm2({L[i * 4 + 2] - L[i * 4 + 0], L[i * 4 + 3] - L[i * 4 + 1]});
            if (len > len_thre) {
                for (int c = 0; c < 4; c++) L[keep * 4 + c] = L[i * 4 + c];
                keep++;
            }
        }
        return keep;
    }
    return total;
}

/* object_3d_util.cpp:380-425 (+ smooth_jump_angles :175-189).  out: 3x2, NaN when no support */
void vp_support_edge_infos(const P2 *vps, const double *mid, const double *edge_angles, int n, double thre12_deg,
                           double thre3_deg, double *out)
{
    for (int i = 0; i < 6; i++) out[i] = std::nan("");
    if (n <= 0) return;
    std::vector<double> raw_inl(n);
    std::vector<int> inl(n);
    for (int vp_id = 0; vp_id < 3; vp_id++) {
        const double thre = (vp_id != 2 ? thre12_deg : thre3_deg) / 180.0 * M_PI;
        int cnt = 0;
        for (int e = 0; e < n; e++) {
            const double raw = ang_atan2(mid[e * 2 + 1] - vps[vp_id].y, mid[e * 2 + 0] - vps[vp_id].x);
            const double nrm = normalize_to_pi(raw);
            double d = std::abs(edge_angles[e] - nrm);
            d = std::min(d, M_PI - d);
            if (d < thre) {
                raw_inl[cnt] = raw;
                inl[cnt] = e;
                cnt++;
            }
        }
        if (cnt > 0) {
            const double base = raw_inl[0];
            int imax = 0, imin = 0;
            double vmax = 0, vmin = 0;
            for (int i = 0; i < cnt; i++) {
                double v = raw_inl[i];
                if ((raw_inl[i] - base) < -M_PI)
                    v = raw_inl[i] + 2 * M_PI;
                else if ((raw_inl[i] - base) > M_PI)
                    v = raw_inl[i] - 2 * M_PI;
                if (i == 0) {
                    vmax = vmin = v;
                } else {
                    if (v > vmax) {
                        vmax = v;
                        imax = i;
                    }
                    if (v < vmin) {
                        vmin = v;
                        imin = i;
                    }
                }
            }
            int low = imax, top = imin;
            if (vp_id > 0) std::swap(low, top);
            out[vp_id * 2 + 0] = edge_angles[inl[low]];
            out[vp_id * 2 + 1] = edge_angles[inl[top]];
        }
    }
}

/* object_3d_util.cpp:427-453.  Clamp of the (latent, inclusive-box) out-of-range index is the
 * build's defined behaviour for the reference's UB (SURVEY.md section 7 "Latent out-of-bounds"). */
double box_edge_sum_dists(const float *dist, int dw, int dh, const P2 *c, const int (*edges)[2], int n_edges, bool reweight)
{
    float sum_dist = 0;
    for (int e = 0; e < n_edges; e++) {
        const P2 c1 = c[edges[e][0]], c2 = c[edges[e][1]];
        for (double s = 0; s < 11; s++) {
            const double px = s / 10.0 * c1.x + (1 - s / 10.0) * c2.x;
            const double py = s / 10.0 * c1.y + (1 - s / 10.0) * c2.y;
            int ix = int(px), iy = int(py);
            ix = std::min(std::max(ix, 0), dw - 1);
            iy = std::min(std::max(iy, 0), dh - 1);
            float d1 = dist[(size_t)iy * dw + ix];
            if (reweight) {
                if (4 <= e && e <= 5) d1 = d1 * 3.0 / 2.0;
                if (6 == e) d1 = d1 * 2.0;
            }
            sum_dist = sum_dist + d1;
        }
    }
    return double(sum_dist);
}

/* object_3d_util.cpp:455-492 */
double box_edge_alignment_angle_error(const double *vp_angles, const int (*ids)[4], const P2 *c)
{
    double total = 0;
    const double not_found_penalty = 30.0 / 180.0 * M_PI * 2;
    for (int vp_id = 0; vp_id < 3; vp_id++) {
        double valid[2];
        int nv = 0;
        for (int i = 0; i < 2; i++)
            if (!std::isnan(vp_angles[vp_id * 2 + i])) valid[nv++] = vp_angles[vp_id * 2 + i];
        if (nv > 0) {
            for (int ee = 0; ee < 2; ee++) {
                const P2 a = c[ids[vp_id][2 * ee]], b = c[ids[vp_id][2 * ee + 1]];
                const double box_edge_angle = normalize_to_pi(ang_atan2(b.y - a.y, b.x - a.x));
                double best = 100;
                for (int i = 0; i < nv; i++) {
                    double t = std::abs(box_edge_angle - valid[i]);
                    t = std::min(t, M_PI - t);
                    if (t < best) best = t;
                }
                total = total + best;
            }
        } else
            total = total + not_found_penalty;
    }
    return total;
}

/* matrix_utils.cpp:316-319 with the tie rule this build defines: ascending value, then ascending index */
void sorted_prefix(const std::vector<double> &v, std::vector<int> &idx, int top_k)
{
    std::partial_sort(idx.begin(), idx.begin() + top_k, idx.end(), [&v](int a, int b) {
        const double va = v[a], vb = v[b];
        const bool na = std::isnan(va), nb = std::isnan(vb);
        if (na || nb) return (!na && nb) || (na == nb && a < b); /* NaN ranks last */
        return va < vb || (va == vb && a < b);
    });
}

/* The one comparison of the path whose outcome can hang on the last bit of a transcendental: `angle_error(cut) > angle_error(cut - 1)`
 * (object_3d_util.cpp:511) between two proposals whose angle errors are mathematically equal (mirror-image configurations) but were summed
 * from atan2 values of different arguments.  Which way it falls depends on the libm of the machine the reference runs on, and it
 * switches between two different kept sets (hence different min-max normalisations).  The oracle records how close the call was
 * (orc_last_cut_margin: smallest relative gap of that comparison over the last orc_detect_cuboid call of this thread) and can be asked
 * to take the other branch when the gap is below 1e-13 (orc_set_cut_flip), so a parity test can tell "the CUDA atan2 rounded one
 * angle the other way" from a real difference. */
static thread_local double g_cut_margin = 1e300;     /* of the box being processed */
static thread_local double g_box_margin[64];          /* per box of the last call (first 64 boxes) */
static thread_local int g_cut_flip = -1, g_cur_box = -1;
extern "C" double orc_last_cut_margin(int box) { return (box >= 0 && box < 64) ? g_box_margin[box] : 1e300; }
extern "C" void orc_set_cut_flip(int box) { g_cut_flip = box; } /* -1: none */

/* Analysis switch, off by default.  With whether_sample_cam_roll_pitch the reference leaves cam_pose at the last pose it set while working
 * on a box and derives the NEXT box's yaw_init from it (box_proposal_detail.cpp:126,237,485): the re-derived yaw is the raw yaw give or
 * take an ulp.  By default the CUDA path starts every box from the raw pose (boxes stay independent; DESIGN.md section 2, "Several boxes
 * in a roll / pitch-sampled frame"; cs_set_profiling bit 10 carries the pose like the reference).  With this switch on the oracle does what
 * the default does, so that tests/test_sampling_deviation.py can count how often the two ways differ and the GPU test can pin the default. */
static thread_local int g_independent_boxes = 0;
extern "C" void orc_set_independent_boxes(int on) { g_independent_boxes = on; }
/* Two more test hooks for the same subject (tests/host_core/carried_emu.cpp lets the oracle stand in for the device under the product's
 * pass structure): the camera yaw the FIRST box of the next call derives its yaw samples from, as if an earlier box had left it (NaN, the
 * default: the pose's own), and the camera yaw the last call left behind after its last box. */
static thread_local double g_first_box_cam_yaw = NAN, g_cam_yaw_left = NAN;
extern "C" void orc_set_first_box_cam_yaw(double yaw) { g_first_box_cam_yaw = yaw; }
extern "C" double orc_cam_yaw_left(void) { return g_cam_yaw_left; }

/* object_3d_util.cpp:495-565 */
void fuse_normalize_scores_v2(const std::vector<double> &dist_error, const std::vector<double> &angle_error,
                              std::vector<double> &combined, std::vector<int> &keep, double weight_vp_angle, bool normalize)
{
    const int n = (int)dist_error.size();
    keep.clear();
    if (n > 4) {
        const int breaking_num = (int)std::round(float(n) / 3.0 * 2.0);
        std::vector<int> ds(n), as;
        std::iota(ds.begin(), ds.end(), 0);
        as = ds;
        sorted_prefix(dist_error, ds, breaking_num);
        sorted_prefix(angle_error, as, breaking_num);
        std::vector<int> dkeep(ds.begin(), ds.begin() + breaking_num - 1);
        const double a_cut = angle_error[as[breaking_num - 1]], a_prev = angle_error[as[breaking_num - 2]];
        bool cut_greater = a_cut > a_prev;
        {
            const double scale = std::max(std::fabs(a_cut), std::fabs(a_prev));
            const double margin = scale > 0 ? std::fabs(a_cut - a_prev) / scale : 0.0;
            if (!std::isnan(margin)) {
                if (margin < g_cut_margin) g_cut_margin = margin; /* an exact tie here can be an inexact one there */
                if (g_cut_flip >= 0 && g_cut_flip == g_cur_box && margin < 1e-13) cut_greater = !cut_greater;
            }
        }
        if (cut_greater) {
            std::vector<int> akeep(as.begin(), as.begin() + breaking_num - 1);
            std::sort(dkeep.begin(), dkeep.end());
            std::sort(akeep.begin(), akeep.end());
            std::set_intersection(dkeep.begin(), dkeep.end(), akeep.begin(), akeep.end(), std::back_inserter(keep));
        } else
            keep = dkeep;
    } else {
        keep.resize(n);
        std::iota(keep.begin(), keep.end(), 0);
    }
    const int m = (int)keep.size();
    double min_d = 1e6, max_d = -1, min_a = 1e6, max_a = -1;
    std::vector<double> dk(m), ak(m);
    for (int i = 0; i < m; i++) {
        const double td = dist_error[keep[i]], ta = angle_error[keep[i]];
        min_d = std::min(min_d, td);
        max_d = std::max(max_d, td);
        min_a = std::min(min_a, ta);
        max_a = std::max(max_a, ta);
        dk[i] = td;
        ak[i] = ta;
    }
    combined.resize(m);
    if (normalize && m > 1) {
        for (int i = 0; i < m; i++) combined[i] = (dk[i] - min_d) / (max_d - min_d);
        if ((max_a - min_a) > 0)
            for (int i = 0; i < m; i++) ak[i] = (ak[i] - min_a) / (max_a - min_a);
        for (int i = 0; i < m; i++) combined[i] = (combined[i] + weight_vp_angle * ak[i]) / (1 + weight_vp_angle);
    } else
        for (int i = 0; i < m; i++) combined[i] = (dk[i] + weight_vp_angle * ak[i]) / (1 + weight_vp_angle);
}

/* object_3d_util.cpp:574-585 (+ ray_plane_interact :568-572) for one pixel */
void plane_hit_3d(const double *T, const double *invK, const double *plane, P2 px, double *world)
{
    double ray[3];
    for (int i = 0; i < 3; i++) ray[i] = (invK[i * 3 + 0] * px.x + invK[i * 3 + 1] * px.y) + invK[i * 3 + 2] * 1.0;
    const double frac = -plane[3] / ((plane[0] * ray[0] + plane[1] * ray[1]) + plane[2] * ray[2]);
    double s[3];
    for (int i = 0; i < 3; i++) s[i] = frac * ray[i];
    double h[4];
    for (int i = 0; i < 4; i++) h[i] = ((T[i * 4 + 0] * s[0] + T[i * 4 + 1] * s[1]) + T[i * 4 + 2] * s[2]) + T[i * 4 + 3] * 1.0;
    for (int i = 0; i < 3; i++) world[i] = h[i] / h[3];
}

/* object_3d_util.cpp:610-648 (+ get_wall_plane_equation :587-600, compute3D_BoxCorner :41-50,
 * similarityTransformation :14-26) */
void change_2d_corner_to_3d_object(const P2 *c, double config_id, double vp_1_position, double yaw_esti,
                                   const double *ground_plane_sensor, const double *T, const double *invK, orc_cuboid &o)
{
    double g[4][3];
    for (int i = 0; i < 4; i++) plane_hit_3d(T, invK, ground_plane_sensor, c[4 + i], g[i]);
    auto dist3 = [](const double *a, const double *b) {
        const double dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
        return std::sqrt((dx * dx + dy * dy) + dz * dz);
    };
    const double length_half = dist3(g[0], g[3]) / 2;
    const double width_half = dist3(g[0], g[1]) / 2;

    /* wall plane through ground points 5-6 */
    const double d[3] = {g[0][0] - g[1][0], g[0][1] - g[1][1], g[0][2] - g[1][2]};
    double nrm[3] = {d[1] * 1.0 - d[2] * 0.0, d[2] * 0.0 - d[0] * 1.0, d[0] * 0.0 - d[1] * 0.0};
    const double nn = std::sqrt((nrm[0] * nrm[0] + nrm[1] * nrm[1]) + nrm[2] * nrm[2]);
    for (int i = 0; i < 3; i++) nrm[i] /= nn;
    const double dist = -((nrm[0] * g[0][0] + nrm[1] * g[0][1]) + nrm[2] * g[0][2]);
    double plane_w[4] = {nrm[0], nrm[1], nrm[2], dist};
    if (dist < 0)
        for (int i = 0; i < 4; i++) plane_w[i] = -plane_w[i];
    double plane_s[4];
    plane_to_sensor(T, plane_w, plane_s);
    double top[3];
    plane_hit_3d(T, invK, plane_s, c[1], top);
    const double height_half = top[2] / 2;

    const double mean_x = (((g[0][0] + g[1][0]) + g[2][0]) + g[3][0]) / 4;
    const double mean_y = (((g[0][1] + g[1][1]) + g[2][1]) + g[3][1]) / 4;

    o.pos[0] = mean_x;
    o.pos[1] = mean_y;
    o.pos[2] = height_half;
    o.rotY = yaw_esti;
    o.scale[0] = length_half;
    o.scale[1] = width_half;
    o.scale[2] = height_half;
    o.box_config_type[0] = config_id;
    o.box_config_type[1] = vp_1_position;
    static const int perm1[8] = {6, 5, 8, 7, 2, 3, 4, 1};
    static const int perm2[8] = {5, 6, 7, 8, 3, 2, 1, 4};
    const int *perm = (vp_1_position == 1) ? perm1 : perm2;
    for (int i = 0; i < 8; i++) {
        o.box_corners_2d[0 * 8 + i] = int(c[perm[i] - 1].x);
        o.box_corners_2d[1 * 8 + i] = int(c[perm[i] - 1].y);
    }
    static const double body[3][8] = {{1, 1, -1, -1, 1, 1, -1, -1}, {1, -1, -1, 1, 1, -1, -1, 1}, {-1, -1, -1, -1, 1, 1, 1, 1}};
    const double cy = std::cos(o.rotY), sy = std::sin(o.rotY);
    const double rot[9] = {cy, -sy, 0, sy, cy, 0, 0, 0, 1};
    double S[16] = {0};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            /* rot * diag(scale): the two zero terms are kept so signed zeros behave as in the product */
            double acc = 0;
            for (int k = 0; k < 3; k++) {
                const double term = rot[i * 3 + k] * (k == j ? o.scale[j] : 0.0);
                acc = (k == 0) ? term : acc + term;
            }
            S[i * 4 + j] = acc;
        }
    S[3] = o.pos[0];
    S[7] = o.pos[1];
    S[11] = o.pos[2];
    S[15] = 1;
    for (int k = 0; k < 8; k++) {
        double h[4];
        for (int i = 0; i < 4; i++)
            h[i] = ((S[i * 4 + 0] * body[0][k] + S[i * 4 + 1] * body[1][k]) + S[i * 4 + 2] * body[2][k]) + S[i * 4 + 3] * 1.0;
        for (int i = 0; i < 3; i++) o.box_corners_3d_world[i * 8 + k] = h[i] / h[3];
    }
}

}  // namespace

/* ====================================================================== OpenCV restatements */

extern "C" void orc_bgr2gray(const uint8_t *bgr, int w, int h, int stride, uint8_t *gray, int gstride, int fixed15)
{
    /* cv::cvtColor(CV_BGR2GRAY) (box_proposal_detail.cpp:64): fixed-point luma.
     * OpenCV >= 4: 15-bit {B 3735, G 19235, R 9798}; OpenCV 2.4/3.x: 14-bit {1868, 9617, 4899}. */
    for (int y = 0; y < h; y++) {
        const uint8_t *s = bgr + (size_t)y * stride;
        uint8_t *d = gray + (size_t)y * gstride;
        for (int x = 0; x < w; x++) {
            const int b = s[3 * x], g = s[3 * x + 1], r = s[3 * x + 2];
            d[x] = fixed15 ? (uint8_t)((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15)
                           : (uint8_t)((b * 1868 + g * 9617 + r * 4899 + (1 << 13)) >> 14);
        }
    }
}

extern "C" void orc_canny(const uint8_t *src, int w, int h, int stride, double low_thresh, double high_thresh, uint8_t *dst)
{
    /* cv::Canny(gray(roi), out, 80, 200) (box_proposal_detail.cpp:197): aperture 3, L1 norm.
     * OpenCV >= 3 re-wraps the source header so an ROI is filtered in isolation (replicated border). */
    if (w <= 0 || h <= 0) return;
    if (low_thresh > high_thresh) std::swap(low_thresh, high_thresh);
    const int low = (int)std::floor(low_thresh), high = (int)std::floor(high_thresh);
    std::vector<int16_t> dx((size_t)w * h), dy((size_t)w * h);
    auto px = [&](int y, int x) -> int {
        y = std::min(std::max(y, 0), h - 1);
        x = std::min(std::max(x, 0), w - 1);
        return src[(size_t)y * stride + x];
    };
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const int gx = (px(y - 1, x + 1) + 2 * px(y, x + 1) + px(y + 1, x + 1)) - (px(y - 1, x - 1) + 2 * px(y, x - 1) + px(y + 1, x - 1));
            const int gy = (px(y + 1, x - 1) + 2 * px(y + 1, x) + px(y + 1, x + 1)) - (px(y - 1, x - 1) + 2 * px(y - 1, x) + px(y - 1, x + 1));
            dx[(size_t)y * w + x] = (int16_t)gx;
            dy[(size_t)y * w + x] = (int16_t)gy;
        }
    /* magnitude with a zero border of one pixel */
    const int mw = w + 2;
    std::vector<int> mag((size_t)mw * (h + 2), 0);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) mag[(size_t)(y + 1) * mw + x + 1] = std::abs((int)dx[(size_t)y * w + x]) + std::abs((int)dy[(size_t)y * w + x]);
    /* map: 0 = weak candidate, 1 = not an edge, 2 = edge; one-pixel border of 1 */
    std::vector<uint8_t> map((size_t)mw * (h + 2), 1);
    std::vector<int> stack;
    const int TG22 = (int)(0.4142135623730950488016887242097 * (1 << 15) + 0.5);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const int *ma = &mag[(size_t)(y + 1) * mw + x + 1];
            const int m = ma[0];
            bool is_max = false;
            if (m > low) {
                const int xs = dx[(size_t)y * w + x], ys = dy[(size_t)y * w + x];
                const int ax = std::abs(xs), ay = std::abs(ys) << 15;
                const int tg22x = ax * TG22;
                if (ay < tg22x) {
                    is_max = (m > ma[-1] && m >= ma[1]);
                } else {
                    const int tg67x = tg22x + (ax << 16);
                    if (ay > tg67x)
                        is_max = (m > ma[-mw] && m >= ma[mw]);
                    else {
                        const int s = (xs ^ ys) < 0 ? -1 : 1;
                        is_max = (m > ma[-mw - s] && m > ma[mw + s]);
                    }
                }
            }
            const size_t mi = (size_t)(y + 1) * mw + x + 1;
            if (is_max) {
                if (m > high) {
                    map[mi] = 2;
                    stack.push_back((int)mi);
                } else
                    map[mi] = 0;
            } else
                map[mi] = 1;
        }
    while (!stack.empty()) {
        const int mi = stack.back();
        stack.pop_back();
        static const int dxy[8][2] = {{-1, -1}, {-1, 0}, {-1, 1}, {0, -1}, {0, 1}, {1, -1}, {1, 0}, {1, 1}};
        for (auto &o : dxy) {
            const int ni = mi + o[0] * mw + o[1];
            if (map[ni] == 0) {
                map[ni] = 2;
                stack.push_back(ni);
            }
        }
    }
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) dst[(size_t)y * w + x] = (map[(size_t)(y + 1) * mw + x + 1] == 2) ? 255 : 0;
}

extern "C" void orc_chamfer_dt(const uint8_t *edges, int w, int h, float *dist)
{
    /* cv::distanceTransform(255 - im_canny, dist, CV_DIST_L2, 3) (box_proposal_detail.cpp:199):
     * two-pass 3x3 chamfer, 16.16 fixed point, a = 0.955, b = 1.3693 (OpenCV C path, non-IPP). */
    if (w <= 0 || h <= 0) return;
    const unsigned HV = (unsigned)std::lrint(0.955f * (1 << 16));
    const unsigned DG = (unsigned)std::lrint(1.3693f * (1 << 16));
    const unsigned DMAX = std::numeric_limits<unsigned>::max() - DG;
    const unsigned INIT = DMAX; /* OpenCV 4.x: border saturates, an edge-free image yields DIST_MAX everywhere */
    const float scale = 1.f / (1 << 16);
    const int step = w + 2;
    std::vector<unsigned> t((size_t)step * (h + 2), INIT);
    for (int i = 0; i < h; i++) {
        unsigned *tmp = &t[(size_t)(i + 1) * step + 1];
        const uint8_t *s = edges + (size_t)i * w;
        for (int j = 0; j < w; j++) {
            if (s[j]) /* edge pixel == zero pixel of (255 - canny) */
                tmp[j] = 0;
            else {
                unsigned t0 = tmp[j - step - 1] + DG;
                unsigned v = tmp[j - step] + HV;
                if (t0 > v) t0 = v;
                v = tmp[j - step + 1] + DG;
                if (t0 > v) t0 = v;
                v = tmp[j - 1] + HV;
                if (t0 > v) t0 = v;
                tmp[j] = (t0 > DMAX) ? DMAX : t0;
            }
        }
    }
    for (int i = h - 1; i >= 0; i--) {
        unsigned *tmp = &t[(size_t)(i + 1) * step + 1];
        float *d = dist + (size_t)i * w;
        for (int j = w - 1; j >= 0; j--) {
            unsigned t0 = tmp[j];
            if (t0 > HV) {
                unsigned v = tmp[j + step + 1] + DG;
                if (t0 > v) t0 = v;
                v = tmp[j + step] + HV;
                if (t0 > v) t0 = v;
                v = tmp[j + step - 1] + DG;
                if (t0 > v) t0 = v;
                v = tmp[j + 1] + HV;
                if (t0 > v) t0 = v;
                tmp[j] = t0;
            }
            t0 = (t0 > DMAX) ? DMAX : t0;
            d[j] = (float)(t0 * scale);
        }
    }
}

extern "C" int orc_merge_break_lines(const double *lines, int n, double dist_thre, double angle_thre_deg, double len_thre, double *out)
{
    std::vector<double> L(lines, lines + (size_t)n * 4);
    const int m = merge_break_lines(L, n, dist_thre, angle_thre_deg, len_thre);
    std::memcpy(out, L.data(), sizeof(double) * 4 * m);
    return m;
}

/* the helpers detect_cuboid calls with its parameters, one call each (flat arrays as oracle/ref/cuboid_ref.cpp's ref_ entry points) */
extern "C" void orc_vp_support_edge_infos(const double *vps, const double *mids, const double *angles, int n, double thre12_deg, double thre3_deg,
                                          double *out)
{
    const P2 v[3] = {{vps[0], vps[1]}, {vps[2], vps[3]}, {vps[4], vps[5]}};
    vp_support_edge_infos(v, mids, angles, n, thre12_deg, thre3_deg, out);
}

extern "C" double orc_box_edge_sum_dists(const float *dist, int dw, int dh, const double *corners16, const int *edges, int n_edges, int reweight)
{
    P2 c[8];
    for (int i = 0; i < 8; i++) c[i] = {corners16[i], corners16[8 + i]};
    return box_edge_sum_dists(dist, dw, dh, c, reinterpret_cast<const int(*)[2]>(edges), n_edges, reweight != 0);
}

extern "C" int orc_fuse_normalize_scores_v2(const double *dist_err, const double *angle_err, int n, double weight_vp_angle, int normalize,
                                            double *combined, int *keep)
{
    std::vector<double> d(dist_err, dist_err + n), a(angle_err, angle_err + n), s;
    std::vector<int> k;
    fuse_normalize_scores_v2(d, a, s, k, weight_vp_angle, normalize != 0);
    for (size_t i = 0; i < k.size(); i++) {
        keep[i] = k[i];
        combined[i] = s[i];
    }
    return (int)k.size();
}

extern "C" int orc_linespace_d(double start, double end, double step, double *out, int cap)
{
    std::vector<double> r;
    linespace<double>(start, end, step, r);
    for (int i = 0; i < (int)r.size() && i < cap; i++) out[i] = r[i];
    return (int)r.size();
}

extern "C" void orc_default_params(orc_params *p)
{
    p->consider_config_1 = 1;
    p->consider_config_2 = 1;
    p->whether_sample_cam_roll_pitch = 0;
    p->whether_sample_bbox_height = 0;
    p->max_cuboid_num = 1;
    p->nominal_skew_ratio = 1;
    p->max_cut_skew = 3;
    p->vp12_edge_angle_thre = 15;
    p->vp3_edge_angle_thre = 10;
    p->shorted_edge_thre = 20;
    p->reweight_edge_distance = 1;
    p->whether_normalize_two_errors = 1;
    p->weight_vp_angle = 0.8;
    p->weight_skew_error = 1.5;
    p->pre_merge_dist_thre = 20;
    p->pre_merge_angle_thre = 5;
    p->edge_length_threshold = 30;
    p->canny_low = 80;
    p->canny_high = 200;
    p->yaw_half_range_deg = 45;
    p->yaw_step_deg = 6;
    p->top_sample_count_override = 0;
}

extern "C" void orc_cam_pose(const double *K, const double *T_wc, double *out13)
{
    CamPose cp;
    std::memcpy(cp.K, K, sizeof(cp.K));
    inv3(cp.K, cp.invK);
    set_cam_pose(cp, T_wc);
    for (int i = 0; i < 3; i++) out13[i] = cp.euler[i];
    for (int i = 0; i < 9; i++) out13[3 + i] = cp.KinvR[i];
    out13[12] = cp.yaw;
}

/* ====================================================================== detect_cuboid */

extern "C" int orc_detect_cuboid(const uint8_t *img, int w, int h, int stride, int channels, const double *K,
                                 const double *T_wc, const double *boxes, int N, const double *lines_in, int M,
                                 const orc_params *pp, int topk_cap, orc_cuboid *out, int *out_counts,
                                 int64_t *n_candidates_total, int64_t *n_valid_total, orc_trace *trace)
{
    g_cut_margin = 1e300;
    const orc_params &p = *pp;
    if (n_candidates_total) *n_candidates_total = 0;
    if (n_valid_total) *n_valid_total = 0;

    CamPose cam;
    std::memcpy(cam.K, K, sizeof(cam.K));
    inv3(cam.K, cam.invK); /* set_calibration :36-40 */
    set_cam_pose(cam, T_wc);
    const CamPose cam_raw = cam;

    /* :62-66 */
    std::vector<uint8_t> gray((size_t)w * h);
    if (channels == 3)
        orc_bgr2gray(img, w, h, stride, gray.data(), w, 1);
    else
        for (int y = 0; y < h; y++) std::memcpy(&gray[(size_t)y * w], img + (size_t)y * stride, w);
    const int img_width = w, img_height = h;

    /* align_left_right_edges :90 (object_3d_util.cpp:147-158) */
    std::vector<double> lines(lines_in, lines_in + (size_t)M * 4);
    for (int i = 0; i < M; i++)
        if (lines[i * 4 + 2] < lines[i * 4 + 0]) {
            std::swap(lines[i * 4 + 0], lines[i * 4 + 2]);
            std::swap(lines[i * 4 + 1], lines[i * 4 + 3]);
        }

    const double ground_plane_world[4] = {0, 0, 1, 0};
    double ground_plane_sensor[4];
    plane_to_sensor(cam.T, ground_plane_world, ground_plane_sensor);

    const bool all_configs[2] = {p.consider_config_1 != 0, p.consider_config_2 != 0};

    for (int b = 0; b < 64; b++) g_box_margin[b] = 1e300;
    for (int object_id = 0; object_id < N; object_id++) {
        g_cur_box = object_id;
        g_cut_margin = 1e300;
        struct MarginKeeper {
            int id;
            ~MarginKeeper()
            {
                if (id < 64) g_box_margin[id] = g_cut_margin;
            }
        } margin_keeper{object_id};
        const double *bb = boxes + (size_t)object_id * 5;
        const int left_x_raw = (int)bb[0];
        const int top_y_raw = (int)bb[1];
        const int obj_width_raw = (int)bb[2];
        const int obj_height_raw = (int)bb[3];
        const int right_x_raw = (int)(left_x_raw + bb[2]);
        const int down_y_raw = top_y_raw + obj_height_raw;
        (void)down_y_raw;

        std::vector<int> down_expand_sample_all;
        down_expand_sample_all.push_back(0);
        if (p.whether_sample_bbox_height) {
            int r = std::max(std::min(20, obj_height_raw - 90), 20);
            r = std::min(r, img_height - top_y_raw - obj_height_raw - 1);
            if (r > 10) down_expand_sample_all.push_back((int)std::round(r / 2));
            down_expand_sample_all.push_back(r);
        }

        if (g_independent_boxes && object_id > 0) { /* analysis only: what the CUDA path does */
            cam = cam_raw;
            plane_to_sensor(cam.T, ground_plane_world, ground_plane_sensor);
        }
        const double cam_yaw_now = (object_id == 0 && !std::isnan(g_first_box_cam_yaw)) ? g_first_box_cam_yaw : cam.yaw;
        const double yaw_init = cam_yaw_now - 90.0 / 180.0 * M_PI;
        std::vector<double> obj_yaw_samples;
        linespace<double>(yaw_init - p.yaw_half_range_deg / 180.0 * M_PI, yaw_init + p.yaw_half_range_deg / 180.0 * M_PI,
                          p.yaw_step_deg / 180.0 * M_PI, obj_yaw_samples);

        std::vector<orc_cuboid> raw_obj_proposals;

        for (size_t hs = 0; hs < down_expand_sample_all.size(); hs++) {
            const int down_expand_sample = down_expand_sample_all[hs];
            const int obj_height_expan = obj_height_raw + down_expand_sample;
            const int down_y_expan = top_y_raw + obj_height_expan;
            const double obj_diaglength_expan = std::sqrt((double)(obj_width_raw * obj_width_raw + obj_height_expan * obj_height_expan));

            std::vector<int> top_x_samples;
            if (p.top_sample_count_override > 0) {
                /* BASELINE C5 dense sweep: a fixed number of evenly spaced integer top-x samples */
                const int cnt = p.top_sample_count_override;
                const int lo = left_x_raw + 5, hi = right_x_raw - 5;
                for (int i = 0; i < cnt && hi >= lo; i++) top_x_samples.push_back(lo + (int)(((int64_t)(hi - lo) * i) / std::max(cnt - 1, 1)));
            } else {
                const int top_sample_resolution = (int)std::round(std::min(20, obj_width_raw / 10));
                linespace<int>(left_x_raw + 5, right_x_raw - 5, top_sample_resolution, top_x_samples);
            }

            const int e = std::min(std::max(std::min(20, obj_width_raw - 100), 10), std::max(std::min(20, obj_height_expan - 100), 10));
            const int left_x_e = std::max(0, left_x_raw - e);
            const int right_x_e = std::min(img_width - 1, right_x_raw + e);
            const int top_y_e = std::max(0, top_y_raw - e);
            const int down_y_e = std::min(img_height - 1, down_y_expan + e);
            const int height_e = down_y_e - top_y_e;
            const int width_e = right_x_e - left_x_e;
            const P2 e_lt = {(double)left_x_e, (double)top_y_e}, e_rb = {(double)right_x_e, (double)down_y_e};

            const bool tr = trace && trace->want_object == object_id && trace->want_height_sample == (int)hs;

            /* :166-174 */
            std::vector<double> Lin;
            Lin.reserve((size_t)M * 4);
            int inside = 0;
            for (int i = 0; i < M; i++) {
                const P2 a = {lines[i * 4 + 0], lines[i * 4 + 1]}, b = {lines[i * 4 + 2], lines[i * 4 + 3]};
                if (inside_box(a, e_lt, e_rb) && inside_box(b, e_lt, e_rb)) {
                    for (int c = 0; c < 4; c++) Lin.push_back(lines[i * 4 + c]);
                    inside++;
                }
            }
            /* :177-182 */
            const int n_lines = merge_break_lines(Lin, inside, p.pre_merge_dist_thre, p.pre_merge_angle_thre, p.edge_length_threshold);
            /* :185-191 */
            std::vector<double> line_angles(n_lines), mid(2 * (size_t)n_lines);
            for (int i = 0; i < n_lines; i++) {
                line_angles[i] = ang_atan2(Lin[i * 4 + 3] - Lin[i * 4 + 1], Lin[i * 4 + 2] - Lin[i * 4 + 0]);
                mid[i * 2 + 0] = (Lin[i * 4 + 0] + Lin[i * 4 + 2]) / 2;
                mid[i * 2 + 1] = (Lin[i * 4 + 1] + Lin[i * 4 + 3]) / 2;
            }

            /* :195-199 */
            std::vector<uint8_t> canny((size_t)std::max(width_e, 0) * std::max(height_e, 0));
            std::vector<float> dist_map(canny.size());
            if (width_e > 0 && height_e > 0) {
                orc_canny(&gray[(size_t)top_y_e * w + left_x_e], width_e, height_e, w, p.canny_low, p.canny_high, canny.data());
                orc_chamfer_dt(canny.data(), width_e, height_e, dist_map.data());
            }
            if (tr) {
                trace->roi[0] = left_x_e;
                trace->roi[1] = top_y_e;
                trace->roi[2] = width_e;
                trace->roi[3] = height_e;
                trace->n_lines_roi = inside;
                trace->n_lines_merged = n_lines;
                if (trace->merged_lines)
                    std::memcpy(trace->merged_lines, Lin.data(), sizeof(double) * 4 * std::min(n_lines, trace->cap_lines));
                const size_t npx = std::min(canny.size(), (size_t)std::max(trace->cap_px, 0));
                if (trace->canny) std::memcpy(trace->canny, canny.data(), npx);
                if (trace->dist) std::memcpy(trace->dist, dist_map.data(), npx * sizeof(float));
            }

            /* :211-226 */
            std::vector<double> rows;    /* n x 9 */
            std::vector<double> corners; /* n x 16 */
            std::vector<int> cand_idx;
            std::vector<double> cam_roll_samples, cam_pitch_samples;
            if (p.whether_sample_cam_roll_pitch) {
                linespace<double>(cam_raw.euler[0] - 6.0 / 180.0 * M_PI, cam_raw.euler[0] + 6.0 / 180.0 * M_PI, 3.0 / 180.0 * M_PI, cam_roll_samples);
                linespace<double>(cam_raw.euler[1] - 6.0 / 180.0 * M_PI, cam_raw.euler[1] + 6.0 / 180.0 * M_PI, 3.0 / 180.0 * M_PI, cam_pitch_samples);
            } else {
                cam_roll_samples.push_back(cam_raw.euler[0]);
                cam_pitch_samples.push_back(cam_raw.euler[1]);
            }

            int cand_counter = 0;
            const int n_top = (int)top_x_samples.size();
            /* :229-465 */
            for (size_t ri = 0; ri < cam_roll_samples.size(); ri++)
                for (size_t pi = 0; pi < cam_pitch_samples.size(); pi++)
                    for (size_t yi = 0; yi < obj_yaw_samples.size(); yi++) {
                        if (p.whether_sample_cam_roll_pitch) {
                            double Tn[16];
                            std::memcpy(Tn, T_wc, sizeof(Tn));
                            double Rn[9];
                            euler_zyx_to_rot(cam_roll_samples[ri], cam_pitch_samples[pi], cam_raw.euler[2], Rn);
                            for (int i = 0; i < 3; i++)
                                for (int j = 0; j < 3; j++) Tn[i * 4 + j] = Rn[i * 3 + j];
                            set_cam_pose(cam, Tn);
                            plane_to_sensor(cam.T, ground_plane_world, ground_plane_sensor);
                        }
                        const double obj_yaw_esti = obj_yaw_samples[yi];
                        P2 vps[3];
                        vanishing_points(cam.KinvR, obj_yaw_esti, vps[0], vps[1], vps[2]);
                        double vp_angles[6];
                        vp_support_edge_infos(vps, mid.data(), line_angles.data(), n_lines, p.vp12_edge_angle_thre, p.vp3_edge_angle_thre, vp_angles);
                        const P2 vp_1 = vps[0], vp_2 = vps[1], vp_3 = vps[2];

                        for (int ti = 0; ti < n_top; ti++) {
                            const int cand_base = cand_counter;
                            cand_counter += 2;
                            const P2 c1 = {(double)top_x_samples[ti], (double)top_y_raw};
                            int vp_1_position = 0;
                            P2 c2 = seg_hit_boundary(vp_1, c1, right_x_raw, top_y_raw, right_x_raw, down_y_expan);
                            if (c2.x == -1) {
                                c2 = seg_hit_boundary(vp_1, c1, left_x_raw, top_y_raw, left_x_raw, down_y_expan);
                                if (c2.x != -1) vp_1_position = 2;
                            } else
                                vp_1_position = 1;
                            if (!(vp_1_position > 0)) continue;
                            if (norm2(sub(c1, c2)) < p.shorted_edge_thre) continue;

                            for (int config_id = 1; config_id < 3; config_id++) {
                                if (!all_configs[config_id - 1]) continue;
                                P2 c3, c4;
                                if (config_id == 1) {
                                    if (vp_1_position == 1)
                                        c4 = seg_hit_boundary(vp_2, c1, left_x_raw, top_y_raw, left_x_raw, down_y_expan);
                                    else
                                        c4 = seg_hit_boundary(vp_2, c1, right_x_raw, top_y_raw, right_x_raw, down_y_expan);
                                    if (c4.y == -1) continue;
                                    if (norm2(sub(c1, c4)) < p.shorted_edge_thre) continue;
                                    c3 = line_intersect(vp_2, c2, vp_1, c4);
                                    if (!inside_box(c3, {(double)left_x_raw, (double)top_y_raw}, {(double)right_x_raw, (double)down_y_expan})) continue;
                                    if (norm2(sub(c3, c4)) < p.shorted_edge_thre || norm2(sub(c3, c2)) < p.shorted_edge_thre) continue;
                                } else {
                                    if (vp_1_position == 1)
                                        c3 = seg_hit_boundary(vp_2, c2, left_x_raw, top_y_raw, left_x_raw, down_y_expan);
                                    else
                                        c3 = seg_hit_boundary(vp_2, c2, right_x_raw, top_y_raw, right_x_raw, down_y_expan);
                                    if (c3.y == -1) continue;
                                    if (norm2(sub(c2, c3)) < p.shorted_edge_thre) continue;
                                    c4 = line_intersect(vp_1, c3, vp_2, c1);
                                    if (!inside_box(c4, {(double)left_x_raw, (double)top_y_e}, {(double)right_x_raw, (double)down_y_e})) continue;
                                    if (norm2(sub(c3, c4)) < p.shorted_edge_thre || norm2(sub(c4, c1)) < p.shorted_edge_thre) continue;
                                }
                                const P2 c5 = seg_hit_boundary(vp_3, c3, left_x_raw, down_y_expan, right_x_raw, down_y_expan);
                                if (c5.y == -1) continue;
                                if (norm2(sub(c3, c5)) < p.shorted_edge_thre) continue;
                                const P2 c6 = line_intersect(vp_2, c5, vp_3, c2);
                                if (!inside_box(c6, e_lt, e_rb)) continue;
                                if (norm2(sub(c6, c2)) < p.shorted_edge_thre || norm2(sub(c6, c5)) < p.shorted_edge_thre) continue;
                                const P2 c7 = line_intersect(vp_1, c6, vp_3, c1);
                                if (!inside_box(c7, e_lt, e_rb)) continue;
                                if (norm2(sub(c7, c1)) < p.shorted_edge_thre || norm2(sub(c7, c6)) < p.shorted_edge_thre) continue;
                                const P2 c8 = line_intersect(vp_1, c5, vp_2, c7);
                                if (!inside_box(c8, e_lt, e_rb)) continue;
                                if (norm2(sub(c8, c4)) < p.shorted_edge_thre || norm2(sub(c8, c5)) < p.shorted_edge_thre ||
                                    norm2(sub(c8, c7)) < p.shorted_edge_thre)
                                    continue;

                                const P2 cs[8] = {c1, c2, c3, c4, c5, c6, c7, c8};
                                P2 sh[8];
                                for (int i = 0; i < 8; i++) sh[i] = {cs[i].x - left_x_e, cs[i].y - top_y_e};
                                double sum_dist, angle_err;
                                if (config_id == 1) {
                                    static const int vis[9][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {1, 5}, {2, 4}, {3, 7}, {4, 7}, {4, 5}};
                                    static const int vpe[3][4] = {{0, 1, 7, 4}, {3, 0, 4, 5}, {3, 7, 1, 5}};
                                    sum_dist = box_edge_sum_dists(dist_map.data(), width_e, height_e, sh, vis, 9, false);
                                    angle_err = box_edge_alignment_angle_error(vp_angles, vpe, cs);
                                } else {
                                    static const int vis[7][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {1, 5}, {2, 4}, {4, 5}};
                                    static const int vpe[3][4] = {{0, 1, 2, 3}, {3, 0, 4, 5}, {2, 4, 1, 5}};
                                    sum_dist = box_edge_sum_dists(dist_map.data(), width_e, height_e, sh, vis, 7, p.reweight_edge_distance != 0);
                                    angle_err = box_edge_alignment_angle_error(vp_angles, vpe, cs);
                                }
                                const double r7 = p.whether_sample_cam_roll_pitch ? cam_roll_samples[ri] : cam_raw.euler[0];
                                const double r8 = p.whether_sample_cam_roll_pitch ? cam_pitch_samples[pi] : cam_raw.euler[1];
                                const double row[9] = {(double)config_id, (double)vp_1_position, obj_yaw_esti, (double)ti,
                                                       sum_dist / obj_diaglength_expan, angle_err, (double)down_expand_sample, r7, r8};
                                rows.insert(rows.end(), row, row + 9);
                                for (int r = 0; r < 2; r++)
                                    for (int i = 0; i < 8; i++) corners.push_back(r == 0 ? cs[i].x : cs[i].y);
                                cand_idx.push_back(cand_base + (config_id - 1));
                            }
                        }
                    }

            const int n_valid = (int)cand_idx.size();
            if (n_candidates_total) *n_candidates_total += cand_counter;
            if (n_valid_total) *n_valid_total += n_valid;

            /* :472-475 */
            std::vector<double> de(n_valid), ae(n_valid), normalized_score;
            for (int i = 0; i < n_valid; i++) {
                de[i] = rows[(size_t)i * 9 + 4];
                ae[i] = rows[(size_t)i * 9 + 5];
            }
            std::vector<int> good;
            fuse_normalize_scores_v2(de, ae, normalized_score, good, p.weight_vp_angle, p.whether_normalize_two_errors != 0);

            if (tr) {
                trace->n_candidates = cand_counter;
                trace->n_valid = n_valid;
                const int nv = std::min(n_valid, trace->cap_valid);
                if (trace->rows) std::memcpy(trace->rows, rows.data(), sizeof(double) * 9 * nv);
                if (trace->corners) std::memcpy(trace->corners, corners.data(), sizeof(double) * 16 * nv);
                if (trace->cand_index) std::memcpy(trace->cand_index, cand_idx.data(), sizeof(int32_t) * nv);
                trace->n_kept = (int)good.size();
                const int nk = std::min((int)good.size(), trace->cap_valid);
                if (trace->kept_ids)
                    for (int i = 0; i < nk; i++) trace->kept_ids[i] = good[i];
                if (trace->kept_scores)
                    for (int i = 0; i < nk; i++) trace->kept_scores[i] = normalized_score[i];
            }

            /* :477-514 */
            for (size_t box_id = 0; box_id < good.size(); box_id++) {
                const int raw = good[box_id];
                const double *rw = &rows[(size_t)raw * 9];
                if (p.whether_sample_cam_roll_pitch) {
                    double Tn[16];
                    std::memcpy(Tn, T_wc, sizeof(Tn));
                    double Rn[9];
                    euler_zyx_to_rot(rw[7], rw[8], cam_raw.euler[2], Rn);
                    for (int i = 0; i < 3; i++)
                        for (int j = 0; j < 3; j++) Tn[i * 4 + j] = Rn[i * 3 + j];
                    set_cam_pose(cam, Tn);
                    plane_to_sensor(cam.T, ground_plane_world, ground_plane_sensor);
                }
                orc_cuboid o;
                std::memset(&o, 0, sizeof(o));
                P2 cs[8];
                for (int i = 0; i < 8; i++) cs[i] = {corners[(size_t)raw * 16 + i], corners[(size_t)raw * 16 + 8 + i]};
                change_2d_corner_to_3d_object(cs, rw[0], rw[1], rw[2], ground_plane_sensor, cam.T, cam.invK, o);
                if (o.scale[0] < 0 || o.scale[1] < 0 || o.scale[2] < 0) continue;
                o.rect_detect_2d[0] = left_x_raw;
                o.rect_detect_2d[1] = top_y_raw;
                o.rect_detect_2d[2] = obj_width_raw;
                o.rect_detect_2d[3] = obj_height_raw;
                o.edge_distance_error = rw[4];
                o.edge_angle_error = rw[5];
                o.normalized_error = normalized_score[box_id];
                o.skew_ratio = std::max(o.scale[0], o.scale[1]) / std::min(o.scale[0], o.scale[1]);
                o.down_expand_height = rw[6];
                if (p.whether_sample_cam_roll_pitch) {
                    o.camera_roll_delta = rw[7] - cam_raw.euler[0];
                    o.camera_pitch_delta = rw[8] - cam_raw.euler[1];
                }
                o.proposal_index = raw;
                o.height_sample_id = (int)hs;
                o.valid = 1;
                raw_obj_proposals.push_back(o);
            }
        } /* height samples */

        /* :517-536 */
        const int n_raw = (int)raw_obj_proposals.size();
        const int actual = std::min(std::min(p.max_cuboid_num, n_raw), topk_cap);
        std::vector<double> score(n_raw);
        for (int i = 0; i < n_raw; i++) {
            orc_cuboid &o = raw_obj_proposals[i];
            double skew_error = p.weight_skew_error * std::max(o.skew_ratio - p.nominal_skew_ratio, 0.0);
            if (o.skew_ratio > p.max_cut_skew) skew_error = 100;
            o.combined_score = o.normalized_error + p.weight_skew_error * skew_error;
            score[i] = o.combined_score;
        }
        std::vector<int> order(n_raw);
        std::iota(order.begin(), order.end(), 0);
        if (actual > 0) sorted_prefix(score, order, actual);
        for (int i = 0; i < actual; i++) out[(size_t)object_id * topk_cap + i] = raw_obj_proposals[order[i]];
        out_counts[object_id] = actual;
    }
    g_cam_yaw_left = cam.yaw;
    return 0;
}
