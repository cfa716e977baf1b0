"""Runs the UNMODIFIED reference (pasco.models.*) on the CPU oracle — build container only
(/root/reference does not exist on the GPU box).  Used to (a) prove the oracle presents the
MinkowskiEngine surface PaSCo needs (BASELINE.json configs[0], the 'plumbing' config) and
(b) generate tests/golden fixtures.

    python oracle/tools/run_reference_on_oracle.py --grid 64 64 8 --occ 0.05
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [os.path.join(ROOT, "oracle", "shims"), os.path.join(ROOT, "compat"), "/root/reference", ROOT]

import numpy as np   # noqa: E402
import torch         # noqa: E402


def synthetic_batch(grid, occ, n_infers=1, in_ch=283, n_classes=20, seed=0):
    """SURVEY.md §8d synthetic scene: Bernoulli occupancy, one point per occupied voxel."""
    g = torch.Generator().manual_seed(seed)
    X, Y, Z = grid
    batch = {"in_feats": [], "in_coords": [], "min_Cs": [], "max_Cs": [], "Ts": []}
    for m in range(n_infers):
        o = torch.rand(X, Y, Z, generator=g) < occ
        c = torch.nonzero(o).int()
        batch["in_coords"].append(c)
        batch["in_feats"].append(torch.randn(c.shape[0], in_ch, generator=g))
        batch["min_Cs"].append(torch.tensor([0, 0, 0]))
        batch["max_Cs"].append(torch.tensor([X - 1, Y - 1, Z - 1]))
        batch["Ts"].append(torch.eye(4))
    batch["global_min_Cs"] = torch.tensor([0, 0, 0])
    batch["global_max_Cs"] = torch.tensor([X - 1, Y - 1, Z - 1])
    sem = {}
    for s in (1, 2, 4):
        lab = torch.randint(1, n_classes, (n_infers, X // s, Y // s, Z // s), generator=g)
        lab[torch.rand(lab.shape, generator=g) < 0.9] = 0
        sem[f"1_{s}"] = lab.to(torch.uint8)
    batch["sem_labels"] = sem
    return batch


def build_net(n_infers=1, f=64, heavy_decoder=False, n_classes=20, in_channels=283, num_queries=100):
    from pasco.models.net_panoptic_sparse import Net
    freqs = {f"1_{s}": np.ones(n_classes) for s in (1, 2, 4)}
    torch.manual_seed(0)
    return Net(n_classes=n_classes, class_names=[str(i) for i in range(n_classes)],
               class_weights=torch.ones(n_classes), encoder_dropouts=[0.0] * 3, decoder_dropouts=[0.0] * 3,
               dense3d_dropout=0.0, n_infers=n_infers, class_frequencies=freqs, in_channels=in_channels,
               num_queries=num_queries, f=f, heavy_decoder=heavy_decoder)


def forward(net, batch, test=False, is_predict_panop=True):
    import MinkowskiEngine as ME
    # CylinderFeat.forward asks pt_fea[0].get_device() (-1 on CPU) for randperm's device
    _rp = torch.randperm
    torch.randperm = lambda n, device=None, **k: _rp(n, **k)
    try:
        in_coords, in_feats = net.feat(batch["in_feats"], batch["in_coords"])
    finally:
        torch.randperm = _rp
    in_feat = ME.SparseTensor(in_feats, in_coords.int())
    in_feat = net.augmenter.merge(in_feat)
    return in_feat, net(in_feat, 1, batch["sem_labels"], global_min_coords=batch["global_min_Cs"],
                        global_max_coords=batch["global_max_Cs"], min_Cs=batch["min_Cs"], max_Cs=batch["max_Cs"],
                        Ts=batch["Ts"], is_predict_panop=is_predict_panop, return_ensemble=False, test=test)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, nargs=3, default=[64, 64, 8])
    ap.add_argument("--occ", type=float, default=0.05)
    ap.add_argument("--f", type=int, default=64)
    ap.add_argument("--n_infers", type=int, default=1)
    ap.add_argument("--no-panop", action="store_true")
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    net = build_net(a.n_infers, a.f)
    net.train()
    batch = synthetic_batch(a.grid, a.occ, a.n_infers)
    t0 = time.time()
    with torch.no_grad():
        in_feat, out = forward(net, batch, is_predict_panop=not a.no_panop)
    dt = time.time() - t0
    print(f"input voxels {in_feat.F.shape}, forward {dt:.2f}s on {os.cpu_count()} cores")
    for s, lg in out["sem_logits_at_scales"].items():
        print("scale", s, [tuple(t.F.shape) for t in lg])
    if "panop_predictions" in out:
        p = out["panop_predictions"][0]
        print("query_logits", tuple(p["query_logits"].shape), "voxel_logits", tuple(p["voxel_logits"].F.shape))
