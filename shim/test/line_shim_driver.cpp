/*
 * shim/test/line_shim_driver.cpp -- TEST HARNESS for shim/line_lbd_b200.cpp (not product code).
 *
 * Builds the shim the way a maintainer would -- against the REFERENCE'S OWN class header
 * (line_lbd/include/line_lbd/line_lbd_allclass.h:22-70, from /root/reference) and cv::Mat -- and calls it the way
 * object_slam/src/main_obj.cpp:363-366,428 does: construct a line_lbd_detect, set use_LSD / line_length_thres, call
 * detect_filter_lines(gray, lines_mat).  This image has no OpenCV C++ headers, so cv::Mat is oracle/ref/minicv.hpp (a container
 * stand-in, see that file); the class, the shim and libcubeslam_b200.so are the real things.  The one member the harness defines itself is
 * the constructor: the reference's (line_lbd_allclass.cpp:110-123) also creates the LBD descriptor / matcher objects, which live in
 * reference translation units outside the cuboid path.
 *
 * Built by oracle/Makefile (target `ref`, only where the reference checkout exists) into oracle/_ref/libshim_line.so;
 * tests/test_gpu_shim_runs.py loads it on the GPU box.
 */
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <exception>
#include <vector>

#include "line_lbd/line_lbd_allclass.h"

line_lbd_detect::line_lbd_detect(int numoctaves, float octaveratio) : numoctaves_(numoctaves), octaveratio_(octaveratio)
{
    use_LSD = false;        /* the class defaults, line_lbd_allclass.cpp:121-122 */
    line_length_thres = 50;
}

/* img: h x w x channels bytes.  out: room for cap rows of [x1 y1 x2 y2].  Returns the number of rows of the n x 4 CV_32F matrix the
 * shim's detect_filter_lines produced, or -1 (message on stderr). */
extern "C" int shim_line_detect_filter(const uint8_t *img, int w, int h, int channels, int use_LSD, float line_length_thres, float *out, int cap)
{
    try {
        line_lbd_detect det(1, 2.0f); /* main_obj.cpp:363: line_lbd_detect line_lbd_obj (one octave) */
        det.use_LSD = use_LSD != 0;
        det.line_length_thres = line_length_thres;
        cv::Mat gray(h, w, channels == 3 ? CV_8UC3 : CV_8UC1);
        std::memcpy(gray.data, img, (size_t)w * h * channels);
        cv::Mat lines;
        det.detect_filter_lines(gray, lines);
        if (lines.rows > 0 && (lines.cols != 4 || lines.type() != CV_32FC1)) return -2;
        const int n = lines.rows < cap ? lines.rows : cap;
        if (n) std::memcpy(out, lines.data, sizeof(float) * 4 * (size_t)n);
        return lines.rows;
    } catch (const std::exception &e) {
        fprintf(stderr, "shim_line_detect_filter: %s\n", e.what());
        return -1;
    }
}

/* the descriptor / matcher members of the shim (SURVEY.md section 8 row f4), called as a user of the class would call them.
 * kl_out: cap x {sx, sy, ex, ey, angle, lineLength, response, size} floats + {numOfPixels, class_id} ints (40 bytes, cs_keyline's layout);
 * desc_out: cap x 32 bytes.  mode 0: detect_descrip_lines(gray, keylines, descrips); 1: detect_descrip_lines_octaves, octave 0;
 * 2: detect_descrip_lines(gray, lines_mat, descrips) (end points only).  Returns the number of lines. */
extern "C" int shim_line_detect_descrip(const uint8_t *img, int w, int h, int channels, int use_LSD, float line_length_thres, int mode, void *kl_out,
                                        uint8_t *desc_out, int cap)
{
    struct Rec {
        float sx, sy, ex, ey, angle, len, response, size;
        int32_t npx, class_id;
    };
    try {
        line_lbd_detect det(1, 2.0f);
        det.use_LSD = use_LSD != 0;
        det.line_length_thres = line_length_thres;
        cv::Mat gray(h, w, channels == 3 ? CV_8UC3 : CV_8UC1);
        std::memcpy(gray.data, img, (size_t)w * h * channels);
        std::vector<cv::line_descriptor::KeyLine> kls;
        cv::Mat desc;
        if (mode == 0)
            det.detect_descrip_lines(gray, kls, desc);
        else if (mode == 1) {
            std::vector<std::vector<cv::line_descriptor::KeyLine>> ko;
            std::vector<cv::Mat> dd;
            det.detect_descrip_lines_octaves(gray, ko, dd);
            if (ko.size() != 1 || dd.size() != 1) return -2;
            kls = ko[0];
            desc = dd[0];
        } else {
            cv::Mat lines;
            det.detect_descrip_lines(gray, lines, desc);
            kls.resize((size_t)lines.rows);
            for (int i = 0; i < lines.rows; i++) {
                const float *r = (const float *)lines.data + 4 * i;
                kls[i].startPointX = r[0];
                kls[i].startPointY = r[1];
                kls[i].endPointX = r[2];
                kls[i].endPointY = r[3];
                kls[i].angle = kls[i].lineLength = kls[i].response = kls[i].size = 0;
                kls[i].numOfPixels = 0;
                kls[i].class_id = i;
            }
        }
        const int n = (int)kls.size();
        if (n > 0 && (desc.rows != n || desc.cols != 32 || desc.type() != CV_8UC1)) return -3;
        for (int i = 0; i < n && i < cap; i++) {
            Rec &o = ((Rec *)kl_out)[i];
            o.sx = kls[i].startPointX;
            o.sy = kls[i].startPointY;
            o.ex = kls[i].endPointX;
            o.ey = kls[i].endPointY;
            o.angle = kls[i].angle;
            o.len = kls[i].lineLength;
            o.response = kls[i].response;
            o.size = kls[i].size;
            o.npx = kls[i].numOfPixels;
            o.class_id = kls[i].class_id;
            std::memcpy(desc_out + (size_t)i * 32, desc.data + (size_t)i * 32, 32);
        }
        return n;
    } catch (const std::exception &e) {
        fprintf(stderr, "shim_line_detect_descrip: %s\n", e.what());
        return -1;
    }
}

/* get_line_descriptors(gray, lines_mat, descrips) and match_line_descrip(query, train, good, thres) through the shim */
extern "C" int shim_line_descriptors_of(const uint8_t *img, int w, int h, int channels, const float *lines, int n, uint8_t *desc_out)
{
    try {
        line_lbd_detect det(1, 2.0f);
        cv::Mat gray(h, w, channels == 3 ? CV_8UC3 : CV_8UC1);
        std::memcpy(gray.data, img, (size_t)w * h * channels);
        cv::Mat rows(n, 4, CV_32FC1), desc;
        if (n) std::memcpy(rows.data, lines, sizeof(float) * 4 * (size_t)n);
        det.get_line_descriptors(gray, rows, desc);
        if (desc.rows != n) return -2;
        if (n) std::memcpy(desc_out, desc.data, (size_t)n * 32);
        return n;
    } catch (const std::exception &e) {
        fprintf(stderr, "shim_line_descriptors_of: %s\n", e.what());
        return -1;
    }
}

extern "C" int shim_line_match(const uint8_t *q, int nq, const uint8_t *t, int nt, float thres, int32_t *query_idx, int32_t *train_idx, float *dist)
{
    try {
        line_lbd_detect det(1, 2.0f);
        cv::Mat mq(nq, 32, CV_8UC1), mt(nt, 32, CV_8UC1);
        if (nq) std::memcpy(mq.data, q, (size_t)nq * 32);
        if (nt) std::memcpy(mt.data, t, (size_t)nt * 32);
        std::vector<cv::DMatch> good;
        det.match_line_descrip(mq, mt, good, thres);
        for (size_t i = 0; i < good.size(); i++) {
            query_idx[i] = good[i].queryIdx;
            train_idx[i] = good[i].trainIdx;
            dist[i] = good[i].distance;
        }
        return (int)good.size();
    } catch (const std::exception &e) {
        fprintf(stderr, "shim_line_match: %s\n", e.what());
        return -1;
    }
}

/* the shim's members for a detector with (numoctaves, octaveratio), LSD flavour: mode 0 detect_raw_lines(gray, vector<vector<KeyLine>>),
 * 1 detect_raw_lines(gray, vector<KeyLine>) split by KeyLine::octave, 2 detect_descrip_lines_octaves.  kl_out: octave k's key lines at
 * k * cap, 64 bytes each (cs_keyline_octave's layout: the 40 bytes above, the in-octave ends, the octave); desc_out likewise in 32-byte rows;
 * counts[k] per octave.  Returns the number of octaves (-1: exception, -6: a KeyLine::pt that is not the mid point of its ends). */
extern "C" int shim_lsd_octaves(const uint8_t *img, int w, int h, int channels, int numoctaves, float octaveratio, float line_length_thres, int mode,
                                void *kl_out, uint8_t *desc_out, int32_t *counts, int cap)
{
    struct Rec {
        float sx, sy, ex, ey, angle, len, response, size;
        int32_t npx, class_id;
        float osx, osy, oex, oey;
        int32_t octave, pad_;
    };
    try {
        line_lbd_detect det(numoctaves, octaveratio);
        det.use_LSD = true;
        det.line_length_thres = line_length_thres;
        cv::Mat gray(h, w, channels == 3 ? CV_8UC3 : CV_8UC1);
        std::memcpy(gray.data, img, (size_t)w * h * channels);
        std::vector<std::vector<cv::line_descriptor::KeyLine>> kls;
        std::vector<cv::Mat> descs;
        if (mode == 0)
            det.detect_raw_lines(gray, kls);
        else if (mode == 1) {
            std::vector<cv::line_descriptor::KeyLine> flat;
            det.detect_raw_lines(gray, flat);
            for (const auto &k : flat) {
                if (k.octave >= (int)kls.size()) kls.resize(k.octave + 1);
                kls[k.octave].push_back(k);
            }
        } else
            det.detect_descrip_lines_octaves(gray, kls, descs);
        for (size_t o = 0; o < kls.size(); o++) {
            const int n = (int)kls[o].size();
            if (n > cap) return -7;
            counts[o] = n;
            for (int i = 0; i < n; i++) {
                const cv::line_descriptor::KeyLine &k = kls[o][i];
                if (k.pt.x != (k.endPointX + k.startPointX) / 2 || k.pt.y != (k.endPointY + k.startPointY) / 2) return -6;
                Rec &r = ((Rec *)kl_out)[o * (size_t)cap + i];
                r = Rec{k.startPointX, k.startPointY, k.endPointX, k.endPointY, k.angle, k.lineLength, k.response, k.size, k.numOfPixels, k.class_id,
                        k.sPointInOctaveX, k.sPointInOctaveY, k.ePointInOctaveX, k.ePointInOctaveY, k.octave, 0};
                if (mode == 2) std::memcpy(desc_out + (o * (size_t)cap + i) * 32, descs[o].data + (size_t)i * 32, 32);
            }
        }
        return (int)kls.size();
    } catch (const std::exception &e) {
        fprintf(stderr, "shim_lsd_octaves: %s\n", e.what());
        return -1;
    }
}
