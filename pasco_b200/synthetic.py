"""Synthetic scenes for BASELINE.json's configs (SURVEY.md §8d): Bernoulli occupancy on an X×Y×Z grid,
one point per occupied voxel, N(0,1) point features, identity pose, labels uniform over classes with
p(empty)=0.9.  CPU tensors (pin + copy them yourself); deterministic in `seed`."""
from __future__ import annotations

from typing import Dict, Sequence

import torch


def clustered_occupancy(grid: Sequence[int], occ: float, g: torch.Generator) -> torch.Tensor:
    """Lidar-like occupancy with the same voxel budget as the Bernoulli scene: a noisy ground slab plus random boxes
    (walls, cars, vegetation blobs), thinned or topped up to exactly round(occ·X·Y·Z) voxels (SURVEY.md §8d: the second
    measurement point — real scenes are clustered, so tiles see more neighbours and fewer rows have none)."""
    X, Y, Z = grid
    target = int(round(occ * X * Y * Z))
    dens = torch.zeros(X, Y, Z)
    dens[:, :, max(0, Z // 8 - 1): Z // 8 + 2] = 0.6                                   # ground slab
    n_boxes = max(4, (X * Y) // 600)
    for _ in range(n_boxes):
        sx, sy = int(torch.randint(6, max(7, X // 5), (1,), generator=g)), int(torch.randint(6, max(7, Y // 5), (1,), generator=g))
        sz = int(torch.randint(2, max(3, Z // 2), (1,), generator=g))
        x0, y0 = int(torch.randint(0, X - sx + 1, (1,), generator=g)), int(torch.randint(0, Y - sy + 1, (1,), generator=g))
        z0 = int(torch.randint(0, max(1, Z - sz + 1), (1,), generator=g))
        dens[x0:x0 + sx, y0:y0 + sy, z0:z0 + sz] = torch.maximum(dens[x0:x0 + sx, y0:y0 + sy, z0:z0 + sz], torch.tensor(0.5))
    score = dens + 0.45 * torch.rand(X, Y, Z, generator=g)          # structure first, uniform noise breaks ties / tops up
    thr = torch.topk(score.view(-1), target).values[-1]
    return score >= thr


def make_scene(grid: Sequence[int] = (256, 256, 32), occ: float = 0.10, n_infers: int = 1, in_ch: int = 283,
               n_classes: int = 20, seed: int = 0, n_masks: int = 10, clustered: bool = False) -> Dict:
    g = torch.Generator().manual_seed(seed)
    X, Y, Z = grid
    b: Dict = {"in_feats": [], "in_coords": [], "min_Cs": [], "max_Cs": [], "Ts": []}
    for _ in range(n_infers):
        o = clustered_occupancy(grid, occ, g) if clustered else torch.rand(X, Y, Z, generator=g) < occ
        c = torch.nonzero(o).int()
        b["in_coords"].append(c)
        b["in_feats"].append(torch.randn(c.shape[0], in_ch, generator=g))
        b["min_Cs"].append(torch.tensor([0, 0, 0]))
        b["max_Cs"].append(torch.tensor([X - 1, Y - 1, Z - 1]))
        b["Ts"].append(torch.eye(4))
    b["global_min_Cs"] = torch.tensor([0, 0, 0])
    b["global_max_Cs"] = torch.tensor([X - 1, Y - 1, Z - 1])
    sem = {}
    for s in (1, 2, 4):
        lab = torch.randint(1, n_classes, (n_infers, X // s, Y // s, Z // s), generator=g)
        lab[torch.rand(lab.shape, generator=g) < 0.9] = 0
        sem[f"1_{s}"] = lab.to(torch.uint8)
    b["sem_labels"] = sem
    # instance masks: random boxes (dense bool [n_masks, X, Y, Z]) with a thing/stuff class each
    boxes = []
    for _ in range(n_masks):
        lo = [int(torch.randint(0, d - d // 4, (1,), generator=g)) for d in (X, Y, Z)]
        boxes.append((lo, [min(d, l + max(2, d // 4)) for l, d in zip(lo, (X, Y, Z))]))
    b["mask_boxes"] = boxes
    b["mask_classes"] = torch.randint(1, n_classes, (n_masks,), generator=g)
    return b


def training_batch(scene: Dict, device="cuda") -> Dict:
    """`make_scene`'s output (unchanged) plus the reference's training fields on `device`: sem_labels, semantic_label
    [M, X, Y, Z] (the scale-1 labels), dense mask_label (one {"labels" uint8 [T], "masks" bool [T, X, Y, Z]} per subnet,
    the scene's boxes) and geo_labels["1_1"] (occupancy, float).  Inputs stay on the host."""
    sem = scene["sem_labels"]["1_1"].to(device)
    grid = tuple(sem.shape[1:])
    masks = torch.zeros(len(scene["mask_boxes"]), *grid, dtype=torch.bool)
    for i, (lo, hi) in enumerate(scene["mask_boxes"]):
        masks[i, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = True
    label = {"labels": scene["mask_classes"].to(torch.uint8).to(device), "masks": masks.to(device)}
    return dict(scene, sem_labels={k: v.to(device) for k, v in scene["sem_labels"].items()}, semantic_label=sem,
                geo_labels={"1_1": (sem > 0).float()}, mask_label=[label] * sem.shape[0])
