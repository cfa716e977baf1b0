"""Round-2 golden vectors — BUILD CONTAINER ONLY (runs the UNMODIFIED reference from /root/reference on the CPU oracle).

    python tests/golden/make_golden_r2.py [case ...]

Cases (all: recipe weights of tests/golden/recipe.py, train-mode BatchNorm):
  big_eval     configs[1] scale, 256x256x32 @10 %, M=1, test=True (no caps): canonical coordinate checksums, per-tensor
               sum / abs-sum and a 1/1024 row subsample (sorted-key order) of every output
  big_capped   same scene, test=False: the cap branch of predict_completion_sem_logit (decoder_v3.py:347-392) with a
               DETERMINISTIC keep-set — torch.multinomial is replaced, in the reference process, by "the n largest
               weights, ties by row index" (a valid draw; the engine-side model uses the same rule in the test)
  m3_caps      64x64x8 @5 %, M=3 with the thresholds lowered (occ_thres / agg_occ_thres are plain attributes) so that the
               per-subnet cap, the vote OR and the M>=3 top-k branch (decoder_v3.py:385-392) all trigger; torch.topk
               replaced by the stable "largest votes, ties by row index" (CPU and CUDA top-k break ties differently)
  kitti360_m3  KITTI-360 shape (19 classes, 8-wide point features, train_kitti360.py:115,152) 64x64x8 @8 %, M=3
  heavy        heavy_decoder=True, 64x64x8 @5 %, M=1
  grads        full-network gradients, 64x64x8 @5 %, M=1: loss = sum over outputs of mean(logits^2); norm + subsample
               of the gradient of ~24 named parameters (incl. dense3d, voxel_feats, input_projs)
"""
import json
import os
import sys
import time

import numpy as np
import torch

import make_golden  # noqa: F401  (sets sys.path to the reference, the oracle and the shims)
import parity
from make_golden import HERE
from recipe import fill_state_dict
from run_reference_on_oracle import build_net, forward
from pasco_b200.synthetic import make_scene

GRAD_PARAMS = [
    "feat.PPmodel.1.weight", "unet3d.encoder.enc_in_feats.kernel", "unet3d.encoder.s1.0.net.2.kernel",
    "unet3d.encoder.s1s2.0.net.0.kernel", "unet3d.encoder.s1s2.3.net.5.kernel", "unet3d.encoder.s2s4.0.net.0.kernel",
    "unet3d.encoder.s4s8.5.net.2.kernel", "unet3d.encoder.s4s8.1.bn.weight",
    "unet3d.dense3d.0.a_conv1.0.weight", "unet3d.dense3d.0.a_conv4.0.weight", "unet3d.dense3d.0.res_3.0.weight",
    "unet3d.dense3d.0.bn_4.weight",
    "unet3d.decoder_generative.dec_blocks.0.upsample.net.0.kernel", "unet3d.decoder_generative.dec_blocks.0.resize.1.kernel",
    "unet3d.decoder_generative.dec_blocks.1.process.1.net.5.kernel", "unet3d.decoder_generative.dec_blocks.2.process.2.net.2.kernel",
    "unet3d.decoder_generative.dec_blocks.2.completion_heads.0.0.kernel", "unet3d.decoder_generative.dec_blocks.2.resize.0.bn.bias",
    "unet3d.decoder_generative.voxel_feats.scale4_infer0.0.kernel", "unet3d.decoder_generative.voxel_feats.scale1_infer0.3.kernel",
    "transformer_predictor.input_projs.0.weight", "transformer_predictor.input_projs.2.weight",
    "transformer_predictor.mask_feat_proj.weight", "transformer_predictor.transformer_cross_attention_layers.1.multihead_attn.in_proj_weight",
    "transformer_predictor.query_feat.weight", "transformer_predictor.mask_embed.layers.2.weight",
]


def _caller_coords(names):
    """Coordinates of the rows being ranked, read from the calling frame of the reference's
    predict_completion_sem_logit (decoder_v3.py:319-394: `sem_logit` / `x` are SparseTensors over those rows)."""
    f = sys._getframe(2)
    for nm in names:
        st = f.f_locals.get(nm)
        if st is not None and hasattr(st, "C"):
            return st.C
    raise RuntimeError("deterministic sampling: caller frame has no coordinates")


def largest_by_value_then_key(w, n, C):
    """The n largest entries of w, ties broken by the packed coordinate key of the row (NOT by the row index: row order
    is implementation-defined, and large regions of a generated scene carry bit-identical features)."""
    order = torch.argsort(parity.keys(C), stable=True)
    rank = torch.sort(w.detach().cpu()[order], descending=True, stable=True)[1][:n]
    return order[rank].to(w.device)


def det_multinomial(w, n, replacement=False, **_):
    """Deterministic stand-in for torch.multinomial(w, n) inside the reference process."""
    return largest_by_value_then_key(w, n, _caller_coords(("sem_logit",)))


def det_topk(x, k, dim=0, **_):
    i = largest_by_value_then_key(x, k, _caller_coords(("x", "sem_logit")))
    return x[i], i


def run_case(tag, grid, occ, n_infers=1, test=False, det=False, heavy=False, n_classes=20, in_ch=283, step=8,
             thresholds=None, grads=False, seed=0):
    t0 = time.time()
    net = build_net(n_infers, 64, heavy_decoder=heavy, n_classes=n_classes, in_channels=in_ch)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.train()
    dec = net.unet3d.decoder_generative
    if thresholds:
        dec.occ_thres, dec.agg_occ_thres = dict(thresholds["occ"]), dict(thresholds["agg"])
    batch = make_scene(grid, occ, n_infers, in_ch=in_ch, n_classes=n_classes, seed=seed)
    saved = (torch.multinomial, torch.topk)
    if det:
        torch.multinomial, torch.topk = det_multinomial, det_topk
    try:
        with torch.set_grad_enabled(grads):
            _, out = forward(net, batch, test=test)
    finally:
        torch.multinomial, torch.topk = saved
    arrays = {}
    parity.collect(out, n_infers, step, arrays, parity.summary)
    meta = {"grid": list(grid), "occ": occ, "seed": seed, "row_step": step, "n_infers": n_infers, "test": test,
            "deterministic_sampling": det, "heavy_decoder": heavy, "n_classes": n_classes, "in_channels": in_ch,
            "thresholds": thresholds}
    if grads:
        loss = 0.0
        for m in range(n_infers):
            for s, lg in out["sem_logits_at_scales"].items():
                loss = loss + lg[m].F.square().mean()
            p = out["panop_predictions"][m]
            loss = loss + p["voxel_logits"].F.square().mean() + p["query_logits"].square().mean()
            for aux in p["aux_outputs"]:
                loss = loss + aux["voxel_logits"].F.square().mean() + aux["query_logits"].square().mean()
        loss.backward()
        arrays["loss"] = np.array([float(loss)])
        named = dict(net.named_parameters())
        for n in GRAD_PARAMS:
            g = named[n].grad.detach().flatten()
            st = max(1, g.numel() // 4096)
            arrays[f"grad::{n}::norm"] = np.array([g.double().norm().item(), g.abs().max().item()])
            arrays[f"grad::{n}::sub"] = g[::st].numpy()
        meta["grad_params"] = GRAD_PARAMS
        # conditioning of these gradients: the SAME reference run with the point features perturbed by 1e-6 (relative).
        # ReLU / argmax masks flip, so the deep layers move by ~1e-2 in relative L2 although the outputs move by 3e-6;
        # the GPU test scales its tolerance with this measured sensitivity instead of inventing one number
        ref_g = {n: named[n].grad.detach().flatten().double().clone() for n in GRAD_PARAMS}
        net.zero_grad(set_to_none=True)
        gen = torch.Generator().manual_seed(123)
        b2 = dict(batch)
        b2["in_feats"] = [f * (1 + 1e-6 * torch.randn(f.shape, generator=gen)) for f in batch["in_feats"]]
        _, out2 = forward(net, b2, test=test)
        loss2 = 0.0
        for s_, lg in out2["sem_logits_at_scales"].items():
            loss2 = loss2 + lg[0].F.square().mean()
        p2 = out2["panop_predictions"][0]
        loss2 = loss2 + p2["voxel_logits"].F.square().mean() + p2["query_logits"].square().mean()
        for aux in p2["aux_outputs"]:
            loss2 = loss2 + aux["voxel_logits"].F.square().mean() + aux["query_logits"].square().mean()
        loss2.backward()
        for n in GRAD_PARAMS:
            g2 = named[n].grad.detach().flatten().double()
            arrays[f"grad::{n}::sens"] = np.array([float((g2 - ref_g[n]).norm() / ref_g[n].norm().clamp(min=1e-30))])
        meta["sensitivity_eps"] = 1e-6
    np.savez_compressed(os.path.join(HERE, f"r2_{tag}.npz"), **arrays)
    json.dump(meta, open(os.path.join(HERE, f"r2_{tag}.json"), "w"), indent=0)
    print(f"{tag}: {time.time() - t0:.1f}s", {k: (v.tolist() if v.size <= 3 else v.shape) for k, v in arrays.items() if k.endswith("_n")})


CASES = {
    "big_eval": dict(grid=(256, 256, 32), occ=0.10, test=True, step=1024),
    "big_capped": dict(grid=(256, 256, 32), occ=0.10, test=False, det=True, step=1024),
    "m3_caps": dict(grid=(64, 64, 8), occ=0.05, n_infers=3, det=True, step=16,
                    thresholds={"occ": {4: 150, 2: 1200, 1: 5000}, "agg": {4: 200, 2: 1500, 1: 6000}}),
    "kitti360_m3": dict(grid=(64, 64, 8), occ=0.08, n_infers=3, n_classes=19, in_ch=8, step=16),
    "heavy": dict(grid=(64, 64, 8), occ=0.05, heavy=True, step=8),
    "grads": dict(grid=(64, 64, 8), occ=0.05, grads=True, step=8),
}

if __name__ == "__main__":
    torch.set_num_threads(os.cpu_count())
    for tag in (sys.argv[1:] or list(CASES)):
        run_case(tag, **CASES[tag])
