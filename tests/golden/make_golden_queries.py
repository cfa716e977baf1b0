"""Generates tests/golden/net_cfg1_q200.npz (+ _manifest.json) by running the UNMODIFIED reference
(pasco.models.*) with num_queries=200 on the CPU oracle — BUILD CONTAINER ONLY (the reference checkout is not on
the GPU box).

    python tests/golden/make_golden_queries.py

Same scene and recipe weights as make_golden.py's cfg1 (64×64×8 @5 %, M=1, f=64, train-mode BatchNorm), but 200
queries: two 128-row query blocks in the engine's cross-attention kernels.  The recipe seeds every parameter by its
name, so the backbone, and with it the semantic logits and the voxel coordinates, are cfg1's: the script checks that
against net_cfg1.npz and stores only what the query count changes, to keep the fixture small.  Stored: a row subsample
of the [P, 200] voxel logits (rows of net_cfg1.npz's canonically sorted `vox_C`), checksums over all of its rows, and
the query logits of the final and the three auxiliary levels.
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

NUM_QUERIES = 200
STEP = 128                 # row subsample of the voxel logits (all 200 columns of every sampled row)


def main():
    torch.set_num_threads(os.cpu_count())
    tag = f"cfg1_q{NUM_QUERIES}"
    net = build_net(1, 64, num_queries=NUM_QUERIES)
    sd = net.state_dict()
    net.load_state_dict(fill_state_dict(sd))
    net.train()
    batch = make_scene(GRID, OCC, 1, seed=SEED)
    with torch.no_grad():
        _, out = forward(net, batch)
    here = os.path.dirname(os.path.abspath(__file__))
    cfg1 = np.load(os.path.join(here, "net_cfg1.npz"))
    arrays = {}
    manifest = {k: list(v.shape) for k, v in sd.items()
                if not k.startswith(("unet3d.transformer_predictor.", "unet3d.decoder_generative.transformer_predictor.",
                                     "criterion."))}
    for s, lg in out["sem_logits_at_scales"].items():         # independent of the query count: cfg1's
        sem = {}
        parity.rows(sem, "sem", lg[0].C, lg[0].F, G.STEP)
        assert np.array_equal(sem["sem_C"], cfg1[f"sem{s}_C"]), s
        err = np.abs(sem["sem_F"] - cfg1[f"sem{s}_F"]).max() / np.abs(cfg1[f"sem{s}_F"]).max()
        assert err <= 1e-5, (s, err)             # CPU rounding between runs; the tests allow 1e-3
    parity.collect(out, 1, STEP, arrays, parity.rows)
    assert np.array_equal(arrays["vox_C"], cfg1["vox_C"])
    arrays = {k: v for k, v in arrays.items() if not k.startswith("sem") and k != "vox_C"}
    np.savez_compressed(os.path.join(here, f"net_{tag}.npz"), **arrays)
    json.dump({"grid": GRID, "occ": OCC, "seed": SEED, "row_step": STEP, "n_infers": 1, "num_queries": NUM_QUERIES,
               "coords_and_sem_from": "net_cfg1.npz", "params": manifest}, open(os.path.join(here, f"net_{tag}_manifest.json"), "w"), indent=0)
    print(tag, {k: v.shape for k, v in arrays.items() if k.endswith("_F") or "query" in k})


if __name__ == "__main__":
    main()
