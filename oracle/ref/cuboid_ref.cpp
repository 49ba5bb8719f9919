/*
 * oracle/ref/cuboid_ref.cpp -- CPU ORACLE, TEST INFRASTRUCTURE ONLY: the reference's own detect_3d_cuboid::detect_cuboid, compiled from
 * /root/reference.
 *
 * One translation unit made of the reference's three sources, included from where they lie:
 *   detect_3d_cuboid/src/matrix_utils.cpp, object_3d_util.cpp, box_proposal_detail.cpp
 * with the reference's own headers, against stand-ins for what this image lacks: oracle/ref/minieigen.hpp for Eigen, oracle/ref/minicv.hpp
 * for OpenCV (Canny / distanceTransform / cvtColor forwarded to the oracle's cv2-pinned restatements), empty ROS / profiler headers
 * (oracle/ref/fakeros).  No reference source is copied.  The sampling loops, the configuration logic, every threshold and index, the
 * scoring and ranking are the reference's code; the linear algebra underneath is the stand-in's (see minieigen.hpp for what that means for
 * the last bits of continuous outputs).
 *
 * Entry point: what object_slam/src/main_obj.cpp:354-361,449 does -- construct detect_3d_cuboid, set_calibration, the mode flags,
 * detect_cuboid(image, pose, boxes, lines, out) -- flattened to plain arrays.  ref_detect_cuboid_skew also sets the member max_cut_skew.
 * Below it, one C entry point per free function of the reference that takes one of detect_cuboid's parameters (merge_break_lines,
 * VP_support_edge_infos, box_edge_sum_dists, fuse_normalize_scores_v2, linespace<double>), so each can be pinned on its own.
 */
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <vector>

#include "/root/reference/detect_3d_cuboid/src/matrix_utils.cpp"
#include "/root/reference/detect_3d_cuboid/src/object_3d_util.cpp"
#include "/root/reference/detect_3d_cuboid/src/box_proposal_detail.cpp"

/* flat record per returned cuboid (doubles): pos[3], rotY, scale[3], box_config_type[2], box_corners_2d[16] (2 x 8, row-major),
 * box_corners_3d_world[24] (3 x 8, row-major), rect_detect_2d[4], edge_distance_error, edge_angle_error, normalized_error, skew_ratio,
 * down_expand_height, camera_roll_delta, camera_pitch_delta  = 60 doubles */
enum { REF_CUBOID_DOUBLES = 60 };

extern "C" int ref_detect_cuboid_skew(const uint8_t *img, int w, int h, int channels, const double *K9, const double *T16, const double *boxes,
                                      int n_boxes, const double *lines, int n_lines, const int *flags, double nominal_skew_ratio, double max_cut_skew,
                                      int max_cuboid_num, double *out, int cap_per_box, int *counts);

extern "C" int ref_detect_cuboid(const uint8_t *img, int w, int h, int channels, const double *K9, const double *T16, const double *boxes, int n_boxes,
                                 const double *lines, int n_lines, const int *flags /* consider_config_1, _2, sample_roll_pitch, sample_bbox_height */,
                                 double nominal_skew_ratio, int max_cuboid_num, double *out, int cap_per_box, int *counts)
{
    return ref_detect_cuboid_skew(img, w, h, channels, K9, T16, boxes, n_boxes, lines, n_lines, flags, nominal_skew_ratio, 3.0, max_cuboid_num, out,
                                  cap_per_box, counts);
}

/* ref_detect_cuboid with the class member max_cut_skew (detect_3d_cuboid.h:79) set as well */
extern "C" int ref_detect_cuboid_skew(const uint8_t *img, int w, int h, int channels, const double *K9, const double *T16, const double *boxes,
                                      int n_boxes, const double *lines, int n_lines, const int *flags, double nominal_skew_ratio, double max_cut_skew,
                                      int max_cuboid_num, double *out, int cap_per_box, int *counts)
{
    try {
        detect_3d_cuboid det;
        det.whether_plot_detail_images = false;
        det.whether_plot_final_images = false;
        det.print_details = false;
        Eigen::Matrix3d K;
        for (int i = 0; i < 3; i++)
            for (int j = 0; j < 3; j++) K(i, j) = K9[i * 3 + j];
        det.set_calibration(K);
        det.consider_config_1 = flags[0] != 0;
        det.consider_config_2 = flags[1] != 0;
        det.whether_sample_cam_roll_pitch = flags[2] != 0;
        det.whether_sample_bbox_height = flags[3] != 0;
        det.nominal_skew_ratio = nominal_skew_ratio;
        det.max_cut_skew = max_cut_skew;
        det.max_cuboid_num = max_cuboid_num;
        Eigen::Matrix4d T;
        for (int i = 0; i < 4; i++)
            for (int j = 0; j < 4; j++) T(i, j) = T16[i * 4 + j];
        Eigen::MatrixXd bb(n_boxes, 5), ed(n_lines, 4);
        for (int i = 0; i < n_boxes; i++)
            for (int j = 0; j < 5; j++) bb(i, j) = boxes[i * 5 + j];
        for (int i = 0; i < n_lines; i++)
            for (int j = 0; j < 4; j++) ed(i, j) = lines[i * 4 + j];
        cv::Mat image(h, w, channels == 3 ? CV_8UC3 : CV_8UC1);
        std::memcpy(image.data, img, (size_t)w * h * channels);
        std::vector<ObjectSet> all;
        det.detect_cuboid(image, T, bb, ed, all);
        for (int b = 0; b < n_boxes; b++) {
            const int n = b < (int)all.size() ? (int)all[b].size() : 0;
            counts[b] = n;
            for (int k = 0; k < n && k < cap_per_box; k++) {
                const cuboid *c = all[b][k];
                double *o = out + ((size_t)b * cap_per_box + k) * REF_CUBOID_DOUBLES;
                int q = 0;
                for (int i = 0; i < 3; i++) o[q++] = c->pos(i);
                o[q++] = c->rotY;
                for (int i = 0; i < 3; i++) o[q++] = c->scale(i);
                for (int i = 0; i < 2; i++) o[q++] = c->box_config_type(i);
                for (int i = 0; i < 2; i++)
                    for (int j = 0; j < 8; j++) o[q++] = c->box_corners_2d(i, j);
                for (int i = 0; i < 3; i++)
                    for (int j = 0; j < 8; j++) o[q++] = c->box_corners_3d_world(i, j);
                for (int i = 0; i < 4; i++) o[q++] = c->rect_detect_2d(i);
                o[q++] = c->edge_distance_error;
                o[q++] = c->edge_angle_error;
                o[q++] = c->normalized_error;
                o[q++] = c->skew_ratio;
                o[q++] = c->down_expand_height;
                o[q++] = c->camera_roll_delta;
                o[q++] = c->camera_pitch_delta;
            }
        }
        for (auto &set : all)
            for (cuboid *c : set) delete c;
        return 0;
    } catch (const std::exception &e) {
        fprintf(stderr, "ref_detect_cuboid: %s\n", e.what());
        return -1;
    }
}

/* ---- the reference's free functions that take detect_cuboid's parameters, one call each, flattened to plain arrays ---- */

/* merge_break_lines (object_3d_util.cpp:300): n x 4 lines in, the merged (and length-filtered) rows out; returns their count */
extern "C" int ref_merge_break_lines(const double *lines, int n, double dist_thre, double angle_thre_deg, double len_thre, double *out)
{
    Eigen::MatrixXd in(n, 4), merged;
    for (int i = 0; i < n; i++)
        for (int j = 0; j < 4; j++) in(i, j) = lines[i * 4 + j];
    merge_break_lines(in, merged, dist_thre, angle_thre_deg, len_thre);
    for (int i = 0; i < (int)merged.rows(); i++)
        for (int j = 0; j < 4; j++) out[i * 4 + j] = merged(i, j);
    return (int)merged.rows();
}

/* VP_support_edge_infos (:380): vps 3 x 2, mids n x 2, angles n, thresholds in degrees -> out 3 x 2 (NaN: no support) */
extern "C" void ref_vp_support_edge_infos(const double *vps, const double *mids, const double *angles, int n, double thre12_deg, double thre3_deg,
                                          double *out)
{
    Eigen::MatrixXd V(3, 2), M(n, 2);
    Eigen::VectorXd A(n);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 2; j++) V(i, j) = vps[i * 2 + j];
    for (int i = 0; i < n; i++) {
        M(i, 0) = mids[i * 2 + 0];
        M(i, 1) = mids[i * 2 + 1];
        A(i) = angles[i];
    }
    Eigen::Vector2d thres;
    thres(0) = thre12_deg;
    thres(1) = thre3_deg;
    const Eigen::MatrixXd r = VP_support_edge_infos(V, M, A, thres);
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 2; j++) out[i * 2 + j] = r(i, j);
}

/* box_edge_sum_dists (:427): dist map dh x dw float32, corners 2 x 8 row-major, edges n_edges x 2 corner ids */
extern "C" double ref_box_edge_sum_dists(const float *dist, int dw, int dh, const double *corners16, const int *edges, int n_edges, int reweight)
{
    cv::Mat dm(dh, dw, CV_32FC1);
    std::memcpy(dm.data, dist, sizeof(float) * (size_t)dw * dh);
    Eigen::MatrixXd C(2, 8);
    for (int i = 0; i < 2; i++)
        for (int j = 0; j < 8; j++) C(i, j) = corners16[i * 8 + j];
    Eigen::MatrixXi E(n_edges, 2);
    for (int i = 0; i < n_edges; i++) {
        E(i, 0) = edges[i * 2 + 0];
        E(i, 1) = edges[i * 2 + 1];
    }
    return box_edge_sum_dists(dm, C, E, reweight != 0);
}

/* fuse_normalize_scores_v2 (:495): n errors each -> kept indices (ascending) and their combined scores; returns the kept count */
extern "C" int ref_fuse_normalize_scores_v2(const double *dist_err, const double *angle_err, int n, double weight_vp_angle, int normalize,
                                            double *combined, int *keep)
{
    Eigen::VectorXd D(n), A(n), S;
    for (int i = 0; i < n; i++) {
        D(i) = dist_err[i];
        A(i) = angle_err[i];
    }
    std::vector<int> k;
    fuse_normalize_scores_v2(D, A, S, k, weight_vp_angle, normalize != 0);
    for (size_t i = 0; i < k.size(); i++) {
        keep[i] = k[i];
        combined[i] = S(i);
    }
    return (int)k.size();
}

/* linespace<double> (matrix_utils.cpp:350): the samples, up to cap of them; returns how many the reference makes */
extern "C" int ref_linespace_d(double start, double end, double step, double *out, int cap)
{
    std::vector<double> r;
    linespace<double>(start, end, step, r);
    for (int i = 0; i < (int)r.size() && i < cap; i++) out[i] = r[i];
    return (int)r.size();
}
