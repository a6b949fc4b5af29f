"""Is the last partial round of a persistent convolution launch idle?  Times single launches at two adjacent batches, the smaller
with at most 6 rounds of 128-row tiles over the SMs and the larger with 7:
   python tests/gpu_checks/conv_chain.py [rotate]

The launches (kgb_bench_conv_ex, kgb_bench_conv_boundary) run on the frame layout: (19 + pad) x (19 + pad) rows per 19x19 image,
pad 1, image after image, so a batch of n has ceil(n * 400 / 128) tiles.  The persistent grid has one CTA per SM and every tile does
the same work, so if the CTAs that run a 7th tile run it while the other SMs idle, the smaller batch takes about 6/7 of the larger
one's time; if the tail overlapped with useful work the ratio would be near the ratio of the batches.  The two batches alternate,
3 runs each, CUDA events over 40 launches after 5 warm-up ones per run, cycling through `rotate` buffer sets (default 4, as
conv_layers.py) so that the working set is larger than the 50 MB L2."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import load_library  # noqa: E402

lib = load_library()
rotate = int(sys.argv[1]) if len(sys.argv) > 1 else 4
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                   capture_output=True, text=True)
print("card:", q.stdout.strip() or q.stderr.strip())
sms = torch.cuda.get_device_properties(0).multi_processor_count
P = (19 + 1) * (19 + 1)


def tiles(n):
    return (n * P + 127) // 128


def rounds(n):
    return (tiles(n) + sms - 1) // sms


# the largest batch whose tiles fit in 6 rounds, and the next one
small = max(n for n in range(1, 1024) if tiles(n) <= 6 * sms)
large = small + 1
assert rounds(small) == 6 and rounds(large) == 7, (small, tiles(small), tiles(large))
print(f"{sms} SMs; batch {small}: {tiles(small)} tiles, {rounds(small)} rounds; batch {large}: {tiles(large)} tiles, {rounds(large)} rounds")


def conv(kind):
    def run(n):
        ms = np.zeros(1, np.float32)
        rc = lib.kgb_bench_conv_ex(3, 3, 192, 192, n, 19, 19, 1, kind, rotate, 5, 40, ms.ctypes.data_as(C.POINTER(C.c_float)))
        assert rc == 0, lib.kgb_last_error()
        return float(ms[0]) * 1e3
    return run


def boundary(n):
    ms = np.zeros(1, np.float32)
    rc = lib.kgb_bench_conv_boundary(192, 384, n, 19, 19, 0, 0, 1, rotate, 5, 40, ms.ctypes.data_as(C.POINTER(C.c_float)))
    assert rc == 0, lib.kgb_last_error()
    return float(ms[0]) * 1e3


for name, fn in (("3x3 192->192 kind 1, fp16", conv(1)), ("3x3 192->192 kind 2, fp16", conv(2)),
                 ("boundary 192/384 fused, fp16 streams", boundary)):
    res = {small: [], large: []}
    for _ in range(3):
        for n in (small, large):
            res[n].append(fn(n))
    a, b = np.median(res[small]), np.median(res[large])
    print(f"{name:38s} batch {small}: " + " ".join(f"{v:7.1f}" for v in res[small]) + " us   batch "
          f"{large}: " + " ".join(f"{v:7.1f}" for v in res[large]) + f" us   ratio {a / b:.4f} (6/7 = {6 / 7:.4f}, "
          f"{small}/{large} = {small / large:.4f}), tail {b - a:6.1f} us per launch", flush=True)
q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader"], capture_output=True, text=True)
print("after:", q.stdout.strip())
