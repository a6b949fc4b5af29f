"""Per-layer timing of the b18c384nbt forward's convolutions, each with the fused epilogue it runs with in fp16 mode:
   python tests/gpu_checks/conv_layers.py [batch] [rotate]

Every launch cycles through `rotate` buffer sets (default 4, as bench.py's roofline object), so at batch 256 the timed loop's
working set is larger than the 50 MB L2.  Epilogue kinds (include/kgb200.h kgb_bench_conv_ex): 0 raw fp32 only, 1 BN + mish
-> fp16 operand, 2 + residual stream in place, 3 raw stream + operand, 4 = kind 2 with an fp32 stream (KGB_STREAM_FP32=trunk).
The per-forward sum counts the layers of the default fp16 build (fp16 streams); compare it with perf_nn.py's ms/forward, which
also holds the gpool, head and input kernels."""
import os, sys, ctypes as C
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import load_library
lib = load_library()
n = int(sys.argv[1]) if len(sys.argv) > 1 else 256
rotate = int(sys.argv[2]) if len(sys.argv) > 2 else 4
# k, cin, cout, epilogue kind, launches per forward, name
layers = [(3, 22, 384, 3, 1, "initial conv"),
          (1, 384, 192, 3, 18, "entry 1x1"),
          (3, 192, 192, 1, 31, "inner 3x3, first of unit"),
          (3, 192, 192, 2, 31, "inner 3x3, second of unit"),
          (3, 192, 192, 0, 5, "gpool conv regular|g"),
          (3, 128, 192, 2, 5, "gpool unit second conv"),
          (1, 192, 384, 2, 18, "exit 1x1, fp16 stream"),
          (1, 192, 384, 4, 0, "exit 1x1, fp32 stream"),
          (1, 384, 192, 0, 1, "heads p1|g1|v1")]
P = 20 * 20   # rows per 19x19 image with one pad row / column
tot = floor_tot = 0.0
for k, cin, cout, kind, count, name in layers:
    ms = np.zeros(1, np.float32)
    rc = lib.kgb_bench_conv_ex(k, k, cin, cout, n, 19, 19, 1, kind, rotate, 5, 40, ms.ctypes.data_as(C.POINTER(C.c_float)))
    assert rc == 0, lib.kgb_last_error()
    us = float(ms[0]) * 1e3
    cin_p, cout_p = (cin + 63) // 64 * 64, (cout + 63) // 64 * 64
    flop = 2.0 * k * k * cin * cout * 361 * n
    stream = 4 if kind == 4 else 2
    per_row = cin_p * 2 + {0: cout_p * 4, 1: cout_p * 2, 2: cout_p * (2 * stream + 2), 3: cout_p * 4, 4: cout_p * (2 * stream + 2)}[kind]
    byts = n * P * per_row
    # floors from the H100 SXM data sheet (989 dense fp16 TFLOP/s, 3.35 TB/s HBM3), not reached rates
    floor = max(flop / 989e12, byts / 3.35e12) * 1e6
    print(f"{name:28s} {k}x{k} {cin:4d}->{cout:4d} kind {kind} x{count:2d}: {us:7.1f} us  {flop / us / 1e6:6.1f} TFLOP/s  "
          f"{byts / us / 1e3:6.0f} GB/s  floor {floor:6.1f} us", flush=True)
    tot += us * count
    floor_tot += floor * count
print(f"sum over the b18c384nbt convolutions at batch {n}: {tot / 1e3:.2f} ms per forward (floors {floor_tot / 1e3:.2f} ms)")
