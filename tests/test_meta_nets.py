"""CPU tests of SGF-metadata (human SL) nets: the loader against the reference's PyTorch model exports (tests/golden/
make_torchref_meta_fixtures.py), the reference's loader messages, and the C ABI's kgb_model_info layout."""
import ctypes as C
import gzip
import os
import subprocess

import numpy as np
import pytest

import kg_nn_oracle as orc
import meta_oracle as mo
from conftest import ROOT
from katago_b200 import KGBError, NeuralNet, modelgen, nn_backend

META_CFGS = ["b2c16_meta", "b2c32nbt_meta", "b1c64nbt_meta"]


def _text_twin(golden_dir, cfg, tmp_path):
    path = os.path.join(golden_dir, "models", f"torchref_{cfg}.bin.gz")
    txt = tmp_path / f"torchref_{cfg}.txt.gz"
    txt.write_bytes(gzip.compress(mo.bin_to_text(gzip.decompress(open(path, "rb").read()))))
    return path, str(txt)


@pytest.mark.parametrize("cfg", META_CFGS)
def test_meta_oracle_matches_reference_pytorch_model(golden_dir, cfg):
    d = np.load(os.path.join(golden_dir, f"torchref_{cfg}.npz"))
    m = mo.load_meta_model(os.path.join(golden_dir, "models", f"torchref_{cfg}.bin.gz"))
    sp, gl, meta = d["spatial_nhwc"].astype(np.float32), d["global_"], d["meta"]
    n = sp.shape[0]
    on_board = sp[..., 0].reshape(n, -1) > 0
    tol = 2e-6  # fp32 summation-order noise only, as for the plain torchref nets
    for opt, key in ((0.0, "policy0"), (1.0, "policy_opt")):
        out = mo.get_output(m, sp, gl, meta, None, [opt] * n)
        assert np.abs(out["policy"][:, :361] - d[key][:, :361])[on_board].max() < tol
        assert np.abs(out["policy"][:, 361] - d[key][:, 361]).max() < tol
        assert np.abs(out["value"] - d["value"]).max() < tol
        assert np.abs(out["score_value"] - d["score_value"]).max() < tol
        assert np.abs(out["ownership"] - d["ownership"])[on_board].max() < tol
    # the encoder matters for these outputs: the same net without it is far off
    plain = orc.get_output(mo.without_encoder(m), sp, gl)
    assert np.abs(plain["value"] - d["value"]).max() > 100 * tol
    # metadata feature 86 (board area) is masked by the PyTorch model; the exported mul1 carries the mask as a zero row
    assert not m.encoder.mul1.w[86].any() and m.encoder.mul1.w.any(axis=1).sum() > 100


@pytest.mark.parametrize("cfg", META_CFGS)
def test_meta_nets_load_from_bin_and_text(golden_dir, cfg, tmp_path):
    path, txt = _text_twin(golden_dir, cfg, tmp_path)
    m = mo.load_meta_model(path)
    infos = [NeuralNet.getModelDesc(NeuralNet.loadModelFile(p)) for p in (path, txt)]
    for d in infos:
        assert d["num_input_meta_channels"] == 192
        assert d["trunk_num_channels"] == m.base.trunk_c and d["num_blocks"] == len(m.base.blocks)
        assert d["conv_macs_per_position"] == orc.conv_macs_per_position(m.base)
    assert {k: v for k, v in infos[0].items() if k != "sha256"} == {k: v for k, v in infos[1].items() if k != "sha256"}
    # the text file holds the same weights, float for float
    t = mo.load_meta_model(txt)
    for a, b in ((m.encoder.mul1.w, t.encoder.mul1.w), (m.encoder.bias2.w, t.encoder.bias2.w), (m.encoder.mul3.w, t.encoder.mul3.w),
                 (m.base.initial_matmul.w, t.base.initial_matmul.w), (m.base.ownership_conv.w, t.base.ownership_conv.w)):
        assert np.array_equal(a, b)


def test_meta_net_mac_count_equals_the_reference_loader():
    # the encoder has no convolution: a b18c384nbt with an encoder has the reference-measured 26 139 072 MACs of b18c384nbt (SURVEY.md §0)
    data = modelgen.model_bytes("b18c384nbt", seed=1, meta_channels=384)
    assert orc.conv_macs_per_position(mo.parse_meta_model(data, True).base) == 26139072


def test_non_meta_nets_report_no_meta_channels(tmp_models):
    assert NeuralNet.getModelDesc(NeuralNet.loadModelFile(tmp_models["tiny_nbt"]))["num_input_meta_channels"] == 0


def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


def test_corrupted_encoder_headers_are_refused_with_the_reference_messages(tmp_path):
    good = modelgen.model_bytes("tiny_nbt", seed=3, meta_channels=32)
    NeuralNet.loadModelFile(_write(tmp_path, "good.bin", good))
    # wrong number of metadata inputs (desc.cpp:1582-1586)
    bad = good.replace(b"sgf_metadata_encoder\n192\n", b"sgf_metadata_encoder\n191\n")
    with pytest.raises(KGBError, match=r"sgf_metadata_encoder: number of in channels \(191\) did not match expected \(192\)"):
        NeuralNet.loadModelFile(_write(tmp_path, "inputs.bin", bad))
    # unknown encoder versions (desc.cpp:2519-2527)
    hdr = b"\n1 0 0 0 0 0 0 0\ntrunk\n"
    assert good.count(hdr) == 1
    with pytest.raises(KGBError, match="metaEncoderVersion not implemented, you may need a newer KataGo version, value was: 2"):
        NeuralNet.loadModelFile(_write(tmp_path, "v2.bin", good.replace(hdr, b"\n2 0 0 0 0 0 0 0\ntrunk\n")))
    with pytest.raises(KGBError, match="metaEncoderVersion unexpected value: -1"):
        NeuralNet.loadModelFile(_write(tmp_path, "vneg.bin", good.replace(hdr, b"\n-1 0 0 0 0 0 0 0\ntrunk\n")))
    # mul3 not matching the trunk width (desc.cpp:1739-1745): a 32 -> 48 mul3 in a 64-channel trunk
    head = b"meta.mul3\n32 64\n@BIN@"
    at = good.index(head) + len(head)
    w48 = np.zeros((32, 48), "<f4").tobytes()
    bad = good[:good.index(head)] + b"meta.mul3\n32 48\n@BIN@" + w48 + good[at + 32 * 64 * 4:]
    with pytest.raises(KGBError, match=r"trunk: sgf_metadata_encoder sgfMetadataEncoder.mul3.outChannels \(48\) != trunkNumChannels \(64\)"):
        NeuralNet.loadModelFile(_write(tmp_path, "mul3.bin", bad))


def test_model_info_layout_agrees_between_the_header_and_ctypes(tmp_path):
    """The struct as C++ code compiled against include/kgb200.h lays it out (the boundary-1 TU and the C ABI's CPU mock compile
    against the same header) and as nn_backend's ctypes mirror does."""
    src = tmp_path / "layout.cpp"
    src.write_text('#include "include/kgb200.h"\n#include <cstddef>\n#include <cstdio>\n'
                   'int main() { printf("%zu %zu %zu\\n", sizeof(kgb_model_info), offsetof(kgb_model_info, conv_macs_per_position), '
                   'offsetof(kgb_model_info, num_input_meta_channels)); }\n')
    exe = tmp_path / "layout"
    subprocess.run(["g++", "-std=c++17", "-I", ROOT, str(src), "-o", str(exe)], check=True)
    size, macs, meta = (int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split())
    M = nn_backend._ModelInfo
    assert (size, macs, meta) == (C.sizeof(M), M.conv_macs_per_position.offset, M.num_input_meta_channels.offset)
    assert M._fields_[-1][0] == "num_input_meta_channels"
