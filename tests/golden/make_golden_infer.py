"""Eval-mode golden vectors — BUILD CONTAINER ONLY (runs the UNMODIFIED reference from /root/reference on the CPU oracle).

    python tests/golden/make_golden_infer.py

Inference (`scripts/eval.py`: model.eval(), forward(test=True)) normalises with the running statistics of every
BatchNorm.  The recipe's running statistics (tests/golden/recipe.py) do not match the activations, and after ~40 layers
an eval forward on them is degenerate, so each network is calibrated first:

  1. weights from recipe.py;
  2. every BatchNorm gets momentum = None (cumulative average) and num_batches_tracked = 0, and one train-mode forward
     under no_grad on a calibration scene (seed CALIB_SEED) sets each running statistic to that scene's batch statistic;
  3. all running statistics (small; the weights are not stored) go into the case's npz as `stat::<reference name>`.

Then net.eval() runs with test=True on the net_cfg1 scene at M = 1 and M = 2, and once at benchmark scale (256x256x32
@10 %, M = 1).  Each case is stored as r2_big_eval-style summaries (parity.summary: row count, wrap-around key sum
and xor of the coordinate set, Σ / Σ|·| / max|·| of the features, a row subsample in sorted-key order, the query logits
of all four levels), one file per case: net_cfg1_infer_<case>.npz, case m1 / m2 / big.  The benchmark-scale network is
calibrated on a benchmark-scale scene: activations grow with the occupancy, and statistics from the small scene would
leave its logits in the thousands.
The generator asserts that no eval forward changed a running statistic or num_batches_tracked.
"""
import json
import os
import time

import numpy as np
import torch

import make_golden  # noqa: F401  (sets sys.path to the reference, the oracle and the shims)
import parity
from make_golden import HERE
from recipe import fill_state_dict
from run_reference_on_oracle import build_net, forward
from pasco_b200.synthetic import make_scene

GRID, OCC, SEED, CALIB_SEED = (64, 64, 8), 0.05, 0, 1
BIG_GRID, BIG_OCC = (256, 256, 32), 0.10
# rows of the subsample: every 64th / 128th / 8192nd (the checksums cover every row)
CASES = (("m1", 1, GRID, OCC, 64), ("m2", 2, GRID, OCC, 128), ("big", 1, BIG_GRID, BIG_OCC, 8192))
STAT_SUFFIXES = (".running_mean", ".running_var", ".num_batches_tracked")


def _norms(net):
    return [m for m in net.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]


def _stats(net):
    return {k: v.detach().clone() for k, v in net.state_dict().items() if k.endswith(STAT_SUFFIXES)}


def calibrated_net(n_infers, grid=GRID, occ=OCC):
    net = build_net(n_infers, 64)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    for bn in _norms(net):
        bn.momentum = None
        bn.num_batches_tracked.zero_()
    net.train()
    with torch.no_grad():
        forward(net, make_scene(grid, occ, n_infers, seed=CALIB_SEED), test=True)
    net.eval()
    return net


def eval_forward(net, batch):
    before = _stats(net)
    with torch.no_grad():
        _, out = forward(net, batch, test=True)
    after = _stats(net)
    assert all(torch.equal(before[k], after[k]) for k in before), "the eval forward changed a running statistic"
    return out


def main():
    torch.set_num_threads(os.cpu_count())
    meta = {"calibration_seed": CALIB_SEED, "cases": {}}
    for tag, M, grid, occ, step in CASES:
        t0 = time.time()
        net = calibrated_net(M, grid, occ)
        st = _stats(net)
        names = {k: list(v.shape) for k, v in st.items() if not k.endswith(".num_batches_tracked")}
        assert all(int(v) == 1 for k, v in st.items() if k.endswith(".num_batches_tracked"))
        arrays = {f"stat::{k}": st[k].numpy() for k in names}
        parity.collect(eval_forward(net, make_scene(grid, occ, M, seed=SEED)), M, step, arrays, parity.summary)
        np.savez_compressed(os.path.join(HERE, f"net_cfg1_infer_{tag}.npz"), **arrays)
        meta["cases"][tag] = {"grid": list(grid), "occ": occ, "seed": SEED, "row_step": step, "n_infers": M, "test": True,
                              "deterministic_sampling": False, "heavy_decoder": False, "n_classes": 20,
                              "in_channels": 283, "running_stats": names}
        print(f"{tag}: {time.time() - t0:.1f}s", {k: v.tolist() for k, v in arrays.items() if k.endswith("_n")})
        del net
    json.dump(meta, open(os.path.join(HERE, "net_cfg1_infer_manifest.json"), "w"), indent=0)


if __name__ == "__main__":
    main()
