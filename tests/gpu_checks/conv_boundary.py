"""Timing of one nested-block boundary of b18c384nbt (exit 1x1 192->384 + entry 1x1 384->192), fused into one launch against the
two launches it replaces:
   python tests/gpu_checks/conv_boundary.py [batch] [rotate]

CUDA events over 40 boundaries after 5 warm-up ones, cycling through `rotate` buffer sets (default 4, as conv_layers.py) so that the
working set is larger than the 50 MB L2 at batch 256.  The GB/s are the algorithmic bytes over the time: per row the pair reads the
inner operand, reads and writes the trunk stream, writes and reads back the activated trunk operand, and writes the inner stream
and operand; the fused launch does all of that except the trunk operand's round trip."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import load_library  # noqa: E402

lib = load_library()
n = int(sys.argv[1]) if len(sys.argv) > 1 else 256
rotate = int(sys.argv[2]) if len(sys.argv) > 2 else 4
inner, trunk = 192, 384
rows = n * 20 * 20   # 19x19 images with one pad row / column
for trunk_fp32, inner_fp32, name in ((0, 0, "fp16 streams"), (1, 0, "fp32 trunk stream"), (1, 1, "fp32 streams")):
    ts, ss = (4 if trunk_fp32 else 2), (4 if inner_fp32 else 2)
    common = inner * 2 + trunk * 2 * ts + inner * ss + inner * 2
    bytes_fused = rows * common
    bytes_pair = rows * (common + trunk * 2 * 2)
    res = {}
    for fused in (1, 0):
        ms = np.zeros(1, np.float32)
        rc = lib.kgb_bench_conv_boundary(inner, trunk, n, 19, 19, trunk_fp32, inner_fp32, fused, rotate, 5, 40,
                                         ms.ctypes.data_as(C.POINTER(C.c_float)))
        assert rc == 0, lib.kgb_last_error()
        res[fused] = float(ms[0]) * 1e3
    print(f"{name:18s} batch {n}: fused {res[1]:7.1f} us ({bytes_fused / 1e6:5.0f} MB, {bytes_fused / res[1] / 1e3:5.0f} GB/s)   "
          f"two launches {res[0]:7.1f} us ({bytes_pair / 1e6:5.0f} MB, {bytes_pair / res[0] / 1e3:5.0f} GB/s)   "
          f"saved {res[0] - res[1]:6.1f} us per boundary, {17 * (res[0] - res[1]) / 1e3:5.2f} ms per b18 forward")
