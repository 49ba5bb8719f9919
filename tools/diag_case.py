"""Diagnostic: one synthetic test case through the cuboid path with a given cs_set_profiling flag, stage by stage against the oracle.

    python tools/diag_case.py --seed 12 --flags 0 32
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=12)
    ap.add_argument("--nb", type=int, default=5)
    ap.add_argument("--flags", type=int, nargs="+", default=[0, 32])
    ap.add_argument("--w", type=int, default=640)
    ap.add_argument("--h", type=int, default=480)
    ap.add_argument("--dump", default="")
    ap.add_argument("--kind", default="indoor")
    args = ap.parse_args()
    import cube_slam_b200 as cs
    from cube_slam_b200 import synthetic as S
    from oracle import pyoracle as O
    F = 6
    imgs, Ts, boxes, lines, K = S.make_batch(args.seed, F, args.w, args.h, args.nb, kind=args.kind, poisson=(args.kind == "indoor"))
    dump = {}
    for fl in args.flags:
        ctx = cs.Context(0, args.w, args.h, F, 16, 4096)
        ctx.set_calibration(K)
        ctx.L.cs_set_profiling(ctx.h, fl)
        p = cs.default_params(max_cuboid_num=3)
        ctx.upload(imgs, Ts, boxes, lines, p)
        ctx.run()
        out, counts = ctx.fetch()
        o = 0
        for f in range(F):
            for b in range(len(boxes[f])):
                ref = O.detect_cuboid(imgs[f], K, Ts[f], boxes[f], lines[f], O.default_params(max_cuboid_num=3), trace_object=b)
                tr = ref["trace"]
                roi = ctx.debug_roi(o)
                cand = ctx.debug_candidates(o)
                bad = []
                if not np.array_equal(roi["canny"], tr["canny"]):
                    bad.append("canny(%d px differ)" % int((roi["canny"] != tr["canny"]).sum()))
                if not np.array_equal(roi["dist"], tr["dist"]):
                    bad.append("dist(%d px differ)" % int((roi["dist"] != tr["dist"]).sum()))
                if roi["n_lines_roi"] != tr["n_lines_roi"] or roi["n_lines_merged"] != tr["n_lines_merged"]:
                    bad.append("lines(%d/%d vs %d/%d)" % (roi["n_lines_roi"], roi["n_lines_merged"], tr["n_lines_roi"], tr["n_lines_merged"]))
                elif not np.array_equal(roi["merged_lines"], tr["merged_lines"]):
                    bad.append("merged lines differ")
                vi = np.nonzero(cand["valid"])[0]
                if cand["n"] != tr["n_candidates"] or not np.array_equal(vi, tr["cand_index"]):
                    bad.append("valid set (%d vs %d)" % (len(vi), len(tr["cand_index"])))
                else:
                    de = np.abs(cand["dist_err"][vi] - tr["rows"][:, 4]).max() if len(vi) else 0
                    ae = np.abs(cand["angle_err"][vi] - tr["rows"][:, 5]).max() if len(vi) else 0
                    if de > 1e-9 or ae > 1e-9:
                        bad.append("errors (dist %.3g angle %.3g)" % (de, ae))
                rc = ref["cuboids"][b]
                if counts[o] != len(rc):
                    bad.append("count %d vs %d" % (counts[o], len(rc)))
                for k in range(min(counts[o], len(rc))):
                    g, q = out[o, k], rc[k]
                    if int(g["proposal_index"]) != int(q["proposal_index"]) or abs(float(g["normalized_error"]) - float(q["normalized_error"])) > 1e-9:
                        bad.append("cut margin %.3g" % ref["cut_margin"][b])
                        bad.append("top%d: index %d vs %d, normalized %.9f vs %.9f, skew %.6f vs %.6f, n_valid %d" % (
                            k, g["proposal_index"], q["proposal_index"], g["normalized_error"], q["normalized_error"], g["skew_ratio"], q["skew_ratio"],
                            len(tr["cand_index"])))
                        dump["rows_f%d_b%d_fl%d" % (f, b, fl)] = tr["rows"]
                        dump["gpu_f%d_b%d_fl%d" % (f, b, fl)] = np.array([[out[o, j]["proposal_index"], out[o, j]["normalized_error"], out[o, j]["combined_score"],
                                                                          out[o, j]["edge_distance_error"], out[o, j]["edge_angle_error"], out[o, j]["skew_ratio"]]
                                                                         for j in range(counts[o])])
                        dump["ref_f%d_b%d_fl%d" % (f, b, fl)] = np.array([[q2["proposal_index"], q2["normalized_error"], q2["combined_score"],
                                                                          q2["edge_distance_error"], q2["edge_angle_error"], q2["skew_ratio"]] for q2 in rc])
                print("flags %d frame %d box %d (%s, lines in ROI %d): %s" % (fl, f, b, roi["roi"], roi["n_lines_roi"], ", ".join(bad) if bad else "ok"), flush=True)
                o += 1
        ctx.close()
    if args.dump and dump:
        np.savez(args.dump, **dump)


if __name__ == "__main__":
    main()
