"""Whole nets in fp32-equivalent mode against the float64 oracle (kg_nn_oracle.get_output(..., dtype=np.float64)).

Measured against float64, the three errors separate what test_gpu_nn_parity.py's 1e-3 against the fp32 oracle cannot:
  E32 = max |fp32-equivalent mode - fp64|,  E16 = max |fp16 mode - fp64|,  Eor = max |fp32 oracle - fp64|
over the policy, value, score and ownership outputs.  The split mode computes every product as ah*wh + al*wh + ah*wl from fp16
halves, about 2^-22 relative per operand where fp16 mode is 2^-11.  Its error is not 2^-11 below fp16 mode's, though: the tensor
core's fp32 accumulation truncates toward zero at every 16-channel step (see test_gpu_conv_fp64.py), and split mode makes three
times as many steps.  On an H100 E16 / E32 comes out near 50 on b18c384nbt, 39 on b28c512nbt, 110 on g170 and 200 on mid_nbt,
and E32 is 20-45x Eor.  A lost split term or a dropped lo half of an activated operand puts fp16-sized errors back into the net
and brings E32 to the order of E16.  The assertion E32 <= E16 / 32 needs no absolute tolerance per net.  Its margin is only about
1.6x on b18c384nbt and 1.2x on b28c512nbt, and that is by design: it comes from the truncating accumulation, which sets E32, and
not from a loose reference.  Eor is printed for comparison.
"""
import os

import numpy as np
import pytest

import kg_nn_oracle as orc
from katago_b200 import modelgen
from test_gpu_nn_parity import run_cuda

pytestmark = pytest.mark.gpu

KEYS = ("policy", "value", "score_value", "ownership")


def _err(got, ref):
    return max(float(np.abs(got[k].astype(np.float64) - ref[k]).max()) for k in KEYS)


@pytest.mark.parametrize("net,n,X,sizes", [
    ("b18c384nbt", 8, 19, [(19, 19), (9, 9), (13, 13), (7, 11)] * 2),   # mixed board sizes
    ("b28c512nbt", 8, 19, [(19, 19), (13, 13), (9, 9), (19, 19)] * 2),   # BASELINE config 3's net; its value head has 144 channels
    ("mid_nbt", 9, 19, None),
    ("g170", 4, 19, None),
])
def test_fp32_equivalent_net_against_fp64(tmp_path, tmp_models, golden_dir, net, n, X, sizes):
    if net == "g170":
        path = os.path.join(golden_dir, "models", "g170-b6c96-s175395328-d26788732.bin.gz")
    elif net in tmp_models:
        path = tmp_models[net]
    else:
        path = modelgen.write_model(str(tmp_path / f"{net}.bin"), net, seed=0)
    sp, gl = modelgen.synthetic_inputs(n, X, X, seed=31 + n, board_sizes=sizes)
    sym = (np.arange(n) * 3 + 1) % 8
    m = orc.load_model(path)
    ref64 = orc.get_output(m, sp, gl, sym, dtype=np.float64)
    e_or = _err(orc.get_output(m, sp, gl, sym), ref64)
    e32 = _err(run_cuda(path, sp, gl, sym, None, False, X, X), ref64)
    e16 = _err(run_cuda(path, sp, gl, sym, None, True, X, X), ref64)
    print(f"{net}: E32 {e32:.3g}  E16 {e16:.3g}  Eor {e_or:.3g}  E16/E32 {e16 / max(e32, 1e-30):.3g}")
    assert e32 <= e16 / 32, (e32, e16, e_or)
