"""Generates tests/golden/net_cfg1.npz by running the UNMODIFIED reference (pasco.models.*) on the CPU
oracle — BUILD CONTAINER ONLY (/root/reference is not on the GPU box).

    python tests/golden/make_golden.py

Config = BASELINE.json configs[0] shape (64×64×8 @5 %) but through the full PaSCo forward (Net3D +
MaskPLS transformer, M=1, f=64, train-mode BatchNorm).  Weights come from tests/golden/recipe.py.
Stored: parameter manifest (names + shapes), canonically sorted coordinates of every output, a row
subsample of the features, and global checksums.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, "oracle", "shims"), os.path.join(ROOT, "compat"), "/root/reference", ROOT,
                os.path.join(ROOT, "oracle"), os.path.join(ROOT, "oracle", "tools"), HERE]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import parity  # noqa: E402
from recipe import fill_state_dict  # noqa: E402
from run_reference_on_oracle import build_net, forward  # noqa: E402
from pasco_b200.synthetic import make_scene  # noqa: E402

GRID, OCC, SEED, STEP = (64, 64, 8), 0.05, 0, 8


def make(n_infers, tag, step):
    net = build_net(n_infers, 64)
    sd = net.state_dict()
    net.load_state_dict(fill_state_dict(sd))
    net.train()
    batch = make_scene(GRID, OCC, n_infers, seed=SEED)
    with torch.no_grad():
        _, out = forward(net, batch)
    arrays = {}
    manifest = {k: list(v.shape) for k, v in sd.items()
                if not k.startswith(("unet3d.transformer_predictor.", "unet3d.decoder_generative.transformer_predictor.",
                                     "criterion."))}
    parity.collect(out, n_infers, step, arrays, parity.rows)
    np.savez_compressed(os.path.join(HERE, f"net_{tag}.npz"), **arrays)
    json.dump({"grid": GRID, "occ": OCC, "seed": SEED, "row_step": step, "n_infers": n_infers, "params": manifest},
              open(os.path.join(HERE, f"net_{tag}_manifest.json"), "w"), indent=0)
    print(tag, {k: v.shape for k, v in arrays.items() if k.endswith("_F") or "query" in k})


def main():
    torch.set_num_threads(os.cpu_count())
    make(1, "cfg1", STEP)
    make(2, "cfg1_m2", 32)


if __name__ == "__main__":
    main()
