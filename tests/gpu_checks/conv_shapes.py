"""Per-shape timing of the convolution kernel at the b18c384nbt / b28c512nbt layer shapes:
   python tests/gpu_checks/conv_shapes.py [batch]"""
import os, sys, ctypes as C
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import load_library
lib = load_library()
n = int(sys.argv[1]) if len(sys.argv) > 1 else 256
shapes = [(3, 192, 192, 72, "b18 inner 3x3"), (1, 384, 192, 18, "b18 block entry 1x1"), (1, 192, 384, 18, "b18 block exit 1x1"),
          (3, 22, 384, 1, "b18 first conv"), (3, 192, 128, 5, "b18 gpool regular"), (3, 192, 64, 5, "b18 gpool g"), (1, 384, 192, 1, "b18 heads p1|g1|v1"),
          (3, 256, 256, 0, "b28 inner 3x3"), (1, 512, 256, 0, "b28 entry"), (1, 256, 512, 0, "b28 exit")]
tot = 0.0
for k, cin, cout, count, name in shapes:
    ms = np.zeros(1, np.float32)
    rc = lib.kgb_bench_conv(k, k, cin, cout, n, 19, 19, 1, 5, 40, ms.ctypes.data_as(C.POINTER(C.c_float)))
    assert rc == 0, lib.kgb_last_error()
    us = float(ms[0]) * 1e3
    flop = 2.0 * k * k * cin * cout * 361 * n
    cin_p, cout_p = (cin + 63) // 64 * 64, (cout + 63) // 64 * 64
    byts = n * 400 * (cin_p * 2 + cout_p * 2 + cout_p * 4)   # fp16 in, fp16 act out, fp32 raw out (upper bound: one of the two outputs is optional)
    # floors from the H100 SXM data sheet (989 dense fp16 TFLOP/s, 3.35 TB/s HBM3), not reached rates
    print(f"{name:24s} {k}x{k} {cin:4d}->{cout:4d} x{count:3d}: {us:7.1f} us  {flop / us / 1e6:7.1f} TFLOP/s  tensor floor {flop / 989e12 * 1e6:5.1f} us  hbm floor {byts / 3.35e12 * 1e6:5.1f} us")
    tot += us * count
print(f"sum over b18 layers: {tot / 1e3:.2f} ms")
