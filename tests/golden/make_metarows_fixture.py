"""Generates tests/golden/metarows.npz: SGF-metadata rows as the reference writes them (run HERE, needs the reference build of
oracle/Makefile.ref).

The rows an SGF-metadata (human SL) net takes come from SGFMetadata::fillMetadataRow (neuralnet/sgfmetadata.cpp) on the profile the
humanSLProfile parameter names (SGFMetadata::getProfile), for the player to move and the board area.  tests/cpp/metarows_driver.cpp,
linked against the unmodified reference, prints them; this script records them for several profiles, both players and a few board
areas, so that the tests feed metadata nets real rows instead of random floats.

    rows    [k, 192] float32
    names   [k] profile names ("dummy_warmup" = SGFMetadata::makeDummyWarmupProfile)
    players [k] "b" / "w"
    areas   [k] board areas
    position_spatial [19, 19, 22], position_global [19]: NNInputs::fillRowV7 of the empty 19x19 board, black to move, tromp-taylor
                                                      rules, komi 7.5 (the position gtp's kata-raw-human-nn evaluates after clear_board)
"""
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..", "..")
PROFILES = ["preaz_5k", "preaz_20k", "rank_9d", "rank_1k", "proyear_1990", "proyear_2023", "dummy_warmup"]
AREAS = [361, 169, 81, 91]


def build_driver(directory):
    """tests/cpp/metarows_driver.cpp linked like oracle/Makefile.drivers links the fixture driver (same reference tree, flags and
    libraries)."""
    make = ["make", "-s", "-f", "oracle/Makefile.drivers", "--eval", "print-%: ; @echo $($*)"]
    ref, cxxflags, libs = (subprocess.run(make + [f"print-{v}"], cwd=ROOT, capture_output=True, text=True, check=True).stdout.strip()
                           for v in ("REF", "CXXFLAGS", "LIBS"))
    exe = os.path.join(directory, "metarows_driver")
    subprocess.run(["g++"] + cxxflags.split() + ["-I" + ref, "-o", exe, "tests/cpp/metarows_driver.cpp"] + libs.split(), cwd=ROOT, check=True)
    return exe


def main():
    with tempfile.TemporaryDirectory() as d:
        exe = build_driver(d)
        args = [f"{n}:{p}:{a}" for n in PROFILES for p in "bw" for a in AREAS]
        out = subprocess.run([exe] + args, capture_output=True, text=True, check=True).stdout
        pos = dict((ln.split()[0], np.array([float(x) for x in ln.split()[1:]], np.float32))
                   for ln in subprocess.run([exe, "position", "tromp-taylor", "7.5"], capture_output=True, text=True, check=True).stdout.splitlines())
    names, players, areas, rows = [], [], [], []
    for ln in out.splitlines():
        f = ln.split()
        names.append(f[0]); players.append(f[1]); areas.append(int(f[2]))
        rows.append(np.array([float(x) for x in f[3:]], np.float32))
    rows = np.stack(rows)
    assert rows.shape == (len(args), 192)
    np.savez_compressed(os.path.join(HERE, "metarows.npz"), rows=rows, names=np.array(names), players=np.array(players),
                        areas=np.array(areas, np.int32), position_spatial=pos["spatial"].reshape(19, 19, 22), position_global=pos["global"])
    print(f"metarows.npz: {rows.shape[0]} rows, {len(np.unique(rows, axis=0))} distinct")


if __name__ == "__main__":
    main()
