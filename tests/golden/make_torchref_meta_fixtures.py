"""Generates tests/golden/torchref_<cfg>_meta.npz + tests/golden/models/torchref_<cfg>_meta.bin.gz for SGF-metadata
(human SL) nets (run HERE, needs /root/reference and tests/golden/metarows.npz).

The same independent check as make_torchref_fixtures.py for the reference's `-meta` configs (python/katago/train/modelconfigs.py:
every config plus a metadata encoder of internal width = trunk width): build the reference's PyTorch model, randomise its parameters,
export it with the reference's own exporter and record torch's outputs on seeded position inputs and on real metadata rows
(tests/golden/metarows.npz, rows of a board area that fits each position).  The PyTorch encoder masks metadata feature 86 (the board
area) at run time; the exporter folds that mask into mul1 (export_model_pytorch.py write_metadata_encoder), so these fixtures decide
whether the file alone reproduces it.
"""
import gzip
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

REF = "/root/reference/python"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from katago.train import modelconfigs  # noqa: E402
from katago.train.model_pytorch import Model  # noqa: E402
from katago_b200 import modelgen  # noqa: E402


def meta_rows(sizes, seed):
    """One real metadata row per position, of that position's board area and a profile drawn from `seed`."""
    d = np.load(os.path.join(HERE, "metarows.npz"))
    rng = np.random.default_rng(seed)
    out = []
    for bx, by in sizes:
        cand = np.flatnonzero(d["areas"] == bx * by)
        if len(cand) == 0:   # an area the fixture does not list: the nearest one (the area is feature 86, which the net ignores)
            cand = np.flatnonzero(d["areas"] == d["areas"][np.argmin(np.abs(d["areas"] - bx * by))])
        out.append(d["rows"][rng.choice(cand)])
    return np.stack(out).astype(np.float32)


def make(cfg_name: str, n: int, seed: int, sizes, base=None, override=None):
    torch.manual_seed(seed)
    cfg = dict(modelconfigs.config_of_name[base or cfg_name])
    cfg.update(override or {})
    cfg.setdefault("activation", "relu")   # the model's default (model_pytorch.py:3080), which its MetadataEncoder reads without one
    assert cfg["metadata_encoder"]["meta_encoder_version"] == 1
    model = Model(cfg, 19)
    model.initialize()
    with torch.no_grad():
        for p in model.parameters():
            p.add_(torch.randn_like(p) * (0.05 if p.dim() > 1 else 0.2))
    model.eval()
    tmp = tempfile.mkdtemp()
    ckpt = os.path.join(tmp, "ckpt.ckpt")
    torch.save({"model": model.state_dict(), "config": cfg}, ckpt)
    stem = "torchref_" + cfg_name.replace("-meta", "_meta")
    subprocess.check_call([sys.executable, os.path.join(REF, "export_model_pytorch.py"), "-checkpoint", ckpt, "-export-dir", tmp,
                           "-model-name", "torchref-" + cfg_name, "-filename-prefix", "m"],
                          cwd=REF, stdout=subprocess.DEVNULL)
    os.makedirs(os.path.join(HERE, "models"), exist_ok=True)
    with open(os.path.join(tmp, "m.bin"), "rb") as f, gzip.open(os.path.join(HERE, "models", f"{stem}.bin.gz"), "wb", compresslevel=9) as g:
        g.write(f.read())
    sp, gl = modelgen.synthetic_inputs(n, 19, 19, seed=seed + 100, board_sizes=sizes)
    meta = meta_rows(sizes, seed + 200)
    with torch.no_grad():
        outs = model(torch.from_numpy(np.ascontiguousarray(sp.transpose(0, 3, 1, 2))), torch.from_numpy(gl), torch.from_numpy(meta))
    o = outs[0] if isinstance(outs[0], (tuple, list)) else outs
    policy, value, misc, moremisc, ownership = o[0].numpy(), o[1].numpy(), o[2].numpy(), o[3].numpy(), o[4].numpy()
    np.savez_compressed(os.path.join(HERE, f"{stem}.npz"), spatial_nhwc=sp.astype(np.float16), global_=gl, meta=meta,
                        policy0=policy[:, 0, :], policy_opt=policy[:, 5, :], value=value,
                        score_value=np.concatenate([misc[:, 0:4], moremisc[:, 0:2]], axis=1),
                        ownership=ownership.reshape(n, -1))
    shutil.rmtree(tmp)
    print(cfg_name, "policy range", policy[:, 0].min(), policy[:, 0].max(), "value", value[0])


if __name__ == "__main__":
    make("b2c16-meta", 4, 11, sizes=[(19, 19), (9, 9), (19, 19), (13, 7)])
    # the stock b1c6nbt config has regularC = mid - gpool = 0, which the reference's own C++ loader rejects (desc.cpp:1700-1704);
    # the same nested-bottleneck family with a gpool inner block, as torchref_b2c32nbt
    make("b2c32nbt-meta", 4, 12, sizes=[(19, 19), (19, 19), (11, 11), (13, 13)], base="b1c6nbt-meta",
         override=dict(trunk_num_channels=32, mid_num_channels=16, gpool_num_channels=8,
                       block_kind=[["rconv1", "bottlenest2"], ["rconv2", "bottlenest2gpool"]],
                       p1_num_channels=8, g1_num_channels=8, v1_num_channels=12, v2_size=16,
                       metadata_encoder=dict(meta_encoder_version=1, internal_num_channels=32)))
    # the b5c192nbt family at a third of its width (trunk 64: one full 64-channel tile, no channel padding; encoder 64 wide) and one
    # nested block, so that the random weights stay a small file
    make("b1c64nbt-meta", 3, 13, sizes=[(19, 19), (9, 9), (19, 19)], base="b5c192nbt-meta",
         override=dict(trunk_num_channels=64, mid_num_channels=32, gpool_num_channels=16, block_kind=[["rconv1", "bottlenest2gpool"]],
                       p1_num_channels=16, g1_num_channels=16, v1_num_channels=16, v2_size=32,
                       metadata_encoder=dict(meta_encoder_version=1, internal_num_channels=64)))
