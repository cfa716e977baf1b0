"""Generates tests/golden/net_cfg1_f{32,96}.npz (+ net_cfg1_widths_manifest.json) by running the UNMODIFIED reference
(pasco.models.*) at network widths f = 32 and f = 96 on the CPU oracle — BUILD CONTAINER ONLY (the reference checkout
is not on the GPU box).

    python tests/golden/make_golden_widths.py

Same scene and recipe weights as make_golden.py's cfg1 (64×64×8 @5 %, M=1, train-mode BatchNorm), but the levels have
f, 2f, 4f, 4f channels: at f = 32 the stride-1 level contracts 32 channels, at f = 96 the deep levels and the dense
bottleneck have 384.  The width changes every output, so each fixture holds the canonically sorted coordinates of the
semantic logits of the three scales and of the voxel logits, every STEP-th row of their features, checksums over all
rows, and the query logits of the final and the three auxiliary levels.  The manifest holds the parameter names and
shapes of both widths.
"""
import json
import os

import numpy as np
import torch

import make_golden as G  # noqa: F401  (sets sys.path to the reference, the oracle and the shims)
from make_golden import GRID, OCC, SEED
import parity
from recipe import fill_state_dict
from run_reference_on_oracle import build_net, forward
from pasco_b200.synthetic import make_scene

WIDTHS = (32, 96)
STEP = 32                  # row subsample of the feature arrays


def main():
    torch.set_num_threads(os.cpu_count())
    here = os.path.dirname(os.path.abspath(__file__))
    manifests = {}
    for f in WIDTHS:
        net = build_net(1, f)
        sd = net.state_dict()
        net.load_state_dict(fill_state_dict(sd))
        net.train()
        batch = make_scene(GRID, OCC, 1, seed=SEED)
        with torch.no_grad():
            _, out = forward(net, batch)
        arrays = {}
        parity.collect(out, 1, STEP, arrays, parity.rows)
        np.savez_compressed(os.path.join(here, f"net_cfg1_f{f}.npz"), **arrays)
        manifests[str(f)] = {k: list(v.shape) for k, v in sd.items()
                             if not k.startswith(("unet3d.transformer_predictor.",
                                                  "unet3d.decoder_generative.transformer_predictor.", "criterion."))}
        print(f, {k: v.shape for k, v in arrays.items() if k.endswith("_C") or "query" in k})
    json.dump({"grid": GRID, "occ": OCC, "seed": SEED, "row_step": STEP, "n_infers": 1, "widths": list(WIDTHS),
               "params": manifests}, open(os.path.join(here, "net_cfg1_widths_manifest.json"), "w"), indent=0)


if __name__ == "__main__":
    main()
