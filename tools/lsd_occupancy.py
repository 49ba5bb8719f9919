"""Prints the registers, local memory, shared memory and CTAs per SM of the LSD seed loop (k_lsd_grow_seq) and front end (k_lsd_front), as the
device reports them (cs_debug_lsd_occupancy), and how many seed-loop CTAs fit beside one front-end CTA.

    python tools/lsd_occupancy.py
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FIELDS = ("registers", "local_bytes", "static_smem", "dynamic_smem", "threads", "ctas_per_sm", "carveout_pct")


def main():
    import torch
    import cube_slam_b200 as cs
    from cube_slam_b200 import _lib
    ctx = cs.Context(0, 640, 480, 1, 16, 8192)
    out = np.zeros(14, np.int32)
    ctx.check(ctx.L.cs_debug_lsd_occupancy(ctx.h, _lib.ptr(out, C.c_int32)))
    try:
        print("GPU:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                                     timeout=30).stdout.strip())
    except (OSError, subprocess.SubprocessError):
        pass
    prop = torch.cuda.get_device_properties(0)
    regs_sm = prop.regs_per_multiprocessor
    res = {}
    for i, name in enumerate(("k_lsd_grow_seq", "k_lsd_front")):
        res[name] = dict(zip(FIELDS, (int(v) for v in out[7 * i:7 * i + 7])))
        print(name, " ".join("%s %d" % kv for kv in res[name].items()))
    # beside one front-end CTA: the register file (256-register allocation units per warp) and the SM's shared memory (1 KB reserved per CTA)
    g, f = res["k_lsd_grow_seq"], res["k_lsd_front"]

    def warp_regs(r):
        return (r * 32 + 255) // 256 * 256

    front_regs = warp_regs(f["registers"]) * f["threads"] // 32
    by_regs = (regs_sm - front_regs) // warp_regs(g["registers"])
    smem_sm = prop.shared_memory_per_multiprocessor
    front_smem = f["static_smem"] + f["dynamic_smem"] + 1024
    by_smem = (smem_sm - front_smem) // (g["static_smem"] + g["dynamic_smem"] + 1024)
    print("k_lsd_grow_seq beside one k_lsd_front CTA: %d by registers, %d by shared memory (all %d KB of it), %d by the CTA limit"
          % (by_regs, by_smem, smem_sm // 1024, 32 - 1))


if __name__ == "__main__":
    main()
