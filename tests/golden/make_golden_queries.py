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
from make_golden import GRID, OCC, SEED, canon
from recipe import fill_state_dict
from pasco_b200.synthetic import make_scene

NUM_QUERIES = 200
STEP = 128                 # row subsample of the voxel logits (all 200 columns of every sampled row)


def build_net(num_queries, n_classes=20):
    """oracle/tools/run_reference_on_oracle.build_net with the query count as a parameter."""
    from pasco.models.net_panoptic_sparse import Net
    freqs = {f"1_{s}": np.ones(n_classes) for s in (1, 2, 4)}
    torch.manual_seed(0)
    return Net(n_classes=n_classes, class_names=[str(i) for i in range(n_classes)],
               class_weights=torch.ones(n_classes), encoder_dropouts=[0.0] * 3, decoder_dropouts=[0.0] * 3,
               dense3d_dropout=0.0, n_infers=1, class_frequencies=freqs, in_channels=283,
               num_queries=num_queries, f=64, heavy_decoder=False)


def main():
    from run_reference_on_oracle import forward
    torch.set_num_threads(os.cpu_count())
    tag = f"cfg1_q{NUM_QUERIES}"
    net = build_net(NUM_QUERIES)
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
        c, f = canon(lg[0])
        assert np.array_equal(c, cfg1[f"sem{s}_C"]), s
        err = np.abs(f[::8] - cfg1[f"sem{s}_F"]).max() / np.abs(cfg1[f"sem{s}_F"]).max()
        assert err <= 1e-5, (s, err)             # CPU rounding between runs; the tests allow 1e-3
    p = out["panop_predictions"][0]
    arrays["query_logits"] = p["query_logits"][0].numpy()
    c, f = canon(p["voxel_logits"])
    assert np.array_equal(c, cfg1["vox_C"])
    arrays["vox_F"] = f[::STEP]
    arrays["vox_sum"] = np.array([f.sum(dtype=np.float64), np.abs(f).sum(dtype=np.float64)])
    for i, aux in enumerate(p["aux_outputs"]):
        arrays[f"aux{i}_query_logits"] = aux["query_logits"][0].numpy()
    np.savez_compressed(os.path.join(here, f"net_{tag}.npz"), **arrays)
    json.dump({"grid": GRID, "occ": OCC, "seed": SEED, "row_step": STEP, "n_infers": 1, "num_queries": NUM_QUERIES,
               "coords_and_sem_from": "net_cfg1.npz", "params": manifest}, open(os.path.join(here, f"net_{tag}_manifest.json"), "w"), indent=0)
    print(tag, {k: v.shape for k, v in arrays.items() if k.endswith("_F") or "query" in k})


if __name__ == "__main__":
    main()
