"""Where a chained b18c384nbt forward spends the time the 7th rounds of its convolution launches used to cost:
   python tests/gpu_checks/conv_chain_timeline.py [out_dir]

Kernel intervals from torch.profiler (CUDA activities) for three forwards on one handle:
  serial 256   the ops one at a time with a synchronise after each (kgb_test_forward_serial): every convolution launch alone,
               801 tiles = 7 rounds on 132 SMs                                                                  -> d7[L]
  serial 253   the same with 791 tiles = 6 rounds                                                                -> d6[L]
  chained 256  the graph forward, each convolution that follows another starting while that one still runs
For launch L of the chained forward, its cost is e[L] = end[L] - end[L-1] (the end of the kernel before it in the forward).  A
launch whose tail the next launch fills would cost about d6[L] * 801 / 791, its work without the idle 7th round; a launch the
chain leaves alone costs d7[L].  Reported per class of launch: chained to the one before or not, followed by a chained launch or
not, with the tails (d7 - d6 * 801 / 791) they hold."""
import json
import os
import sys
import tempfile

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from katago_b200 import NeuralNet, load_library, modelgen  # noqa: E402

out_dir = sys.argv[1] if len(sys.argv) > 1 else None
lib = load_library()
lm = NeuralNet.loadModelFile(modelgen.write_model(os.path.join(tempfile.mkdtemp(), "b18.bin"), "b18c384nbt", seed=0))
ctx = NeuralNet.createComputeContext([0], 19, 19, True, lm)
h = NeuralNet.createComputeHandle(ctx, lm, 256, False, True, 0)
dev = torch.device("cuda:0")
bufs = {}


def forward(n, fn):
    if n not in bufs:
        sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=5)
        bufs[n] = [torch.from_numpy(sp.reshape(n, -1)).to(dev), torch.from_numpy(gl).to(dev)] + \
                  [torch.empty((n, w), device=dev) for w in (362, 3, 6, 361)]
    b = bufs[n]
    rc = fn(h._p, n, b[0].data_ptr(), b[1].data_ptr(), None, None, *(x.data_ptr() for x in b[2:]))
    assert rc == 0, lib.kgb_last_error()
    h.sync()


def kernels(n, fn, reps=3):
    """[(name, start_us, end_us)] of the forward's kernels, for the median forward of `reps` by span."""
    for _ in range(2):
        forward(n, fn)
    torch.cuda.synchronize()
    runs = []
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            forward(n, fn)
            torch.cuda.synchronize()
        path = os.path.join(tempfile.mkdtemp(), "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
        ev = sorted((x["name"], float(x["ts"]), float(x["ts"]) + float(x["dur"])) for x in trace["traceEvents"] if x.get("cat") == "kernel")
        ev.sort(key=lambda x: x[1])
        runs.append(ev)
    runs.sort(key=lambda ev: ev[-1][2] - ev[0][1])
    return runs[len(runs) // 2]


is_conv = lambda name: "kgb_conv_wg_kernel" in name or "kgb_conv_pair_kernel" in name
s7 = kernels(256, lib.kgb_test_forward_serial)
s6 = kernels(253, lib.kgb_test_forward_serial)
ch = kernels(256, lib.kgb_forward_device)
assert len(s7) == len(s6) == len(ch), (len(s7), len(s6), len(ch))
assert all(a[0] == b[0] for a, b in zip(s7, ch))
d7 = np.array([e - s for _, s, e in s7])
d6 = np.array([e - s for _, s, e in s6]) * 801.0 / 791.0
conv = np.array([is_conv(k[0]) for k in ch])
end = np.array([k[2] for k in ch])
e = np.diff(np.concatenate([[ch[0][1]], end]))
linked = np.array([i > 0 and conv[i] and conv[i - 1] for i in range(len(ch))])     # chained to the launch before
feeds = np.array([i + 1 < len(ch) and linked[i + 1] for i in range(len(ch))])       # the next launch is chained to it
span = lambda ev: ev[-1][2] - ev[0][1]
print(f"kernels per forward {len(ch)}, convolution launches {conv.sum()}, chained {linked.sum()}")
print(f"forward span: serial 256 {span(s7) / 1e3:.3f} ms (kernels only, gaps from the synchronises included), chained 256 {span(ch) / 1e3:.3f} ms")
print(f"sum of kernel times alone: 256 {d7.sum() / 1e3:.3f} ms (convolutions {d7[conv].sum() / 1e3:.3f}), 253 scaled to 801 tiles "
      f"{d6.sum() / 1e3:.3f} ms (convolutions {d6[conv].sum() / 1e3:.3f})")
print(f"7th-round tails (d7 - d6 * 801/791) of all convolution launches: {(d7 - d6)[conv].sum() / 1e3:.3f} ms")
rows = []
for name, sel in (("conv, feeds a chained launch", conv & feeds), ("conv, the last of a chain", conv & ~feeds),
                  ("other kernels", ~conv)):
    rows.append(dict(cls=name, count=int(sel.sum()), alone_7=float(d7[sel].sum()), alone_6s=float(d6[sel].sum()),
                     tail=float((d7 - d6)[sel].sum())))
    print(f"{name:32s} x{sel.sum():3d}: alone {d7[sel].sum() / 1e3:7.3f} ms, without 7th-round tails {d6[sel].sum() / 1e3:7.3f} ms, "
          f"tails {(d7 - d6)[sel].sum() / 1e3:6.3f} ms")
print(f"chained launches: cost e[L] {e[linked].sum() / 1e3:.3f} ms against alone d7 {d7[linked].sum() / 1e3:.3f} ms; their predecessors' "
      f"tails {(d7 - d6)[np.where(linked)[0] - 1].sum() / 1e3:.3f} ms; saved {(d7[linked] - e[linked]).sum() / 1e3:.3f} ms")
print(f"unchained kernels: cost {e[~linked].sum() / 1e3:.3f} ms against alone {d7[~linked].sum() / 1e3:.3f} ms")
# per chained launch: how much of its predecessor's tail it recovered
rec = (d7[linked] - e[linked]) / np.maximum((d7 - d6)[np.where(linked)[0] - 1], 1e-3)
print("recovered share of the predecessor's tail per chained launch: median %.2f, quartiles %.2f / %.2f, min %.2f" %
      (np.median(rec), np.percentile(rec, 25), np.percentile(rec, 75), rec.min()))
if out_dir:
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "conv_chain_timeline.json"), "w") as f:
        json.dump(dict(rows=rows, kernels=[dict(name=k[0][:60], start=k[1], end=k[2], alone7=float(a), alone6s=float(b), linked=bool(li))
                                           for k, a, b, li in zip(ch, d7, d6, linked)]), f)
h.free()
ctx.free()
