"""Opt-in hooks that route the UNMODIFIED reference's mask-transformer hot spots onto the sm_90a attention kernels, and
(install(postprocess=True)) its test-time post-processing onto the panoptic kernels.

The MinkowskiEngine surface (`pasco_b200.me`) already carries every sparse-tensor op of the reference.  Two pieces of
PaSCo's transformer are plain torch in the reference and therefore outside that surface:

  * `CrossAttentionLayer.forward`  (pasco/models/transformer/blocks.py:73-92): `nn.MultiheadAttention` of 100 queries over
    all P voxels — cuBLAS batched GEMMs + a [8, 100, P] softmax volume;
  * `TransformerPredictorV2.compute_attn_mask` (transformer/transformer_predictor_v2.py:220-289): a dense
    [1, 100, X/s, Y/s, Z/s] volume (839 MB at scale 1) built only to be sampled at the key voxels.

The reference's `TransformerPredictorV2.forward` (transformer_predictor_v2.py:111-218) then repeats that bool mask over
the heads and sums it in int64 (line 164): 37.5 GiB at M = 3 and full scene size.  `install()` replaces that forward
— at run time, on the imported class, without touching the reference's files — with one that calls the reference's own
submodules but builds each level's mask on the device directly as the bit rows the attention kernels read
(ops.attention_mask_bits: an OR-pool of the thresholded logits to the key scale, a hash look-up of the keys, Q·P/8
bytes per item), and `CrossAttentionLayer.forward` with one that takes those bits into ops.cross_attention, which
net3d's own decoder uses too (K/V projections on the wgmma GEMM, the masked softmax·V as
`pasco_xattn_forward/backward`: streaming two-pass softmax, no [Q, P] score volume in HBM).  Same parameters, same
state_dict, same results within the fp32 tolerance (tests/test_dropin_reference.py and tests/test_attn_mask_bits.py
run the reference with and without the hooks).

The post-processing hooks replace `Ensembler.ensemble_sem_compl` / `ensemble_panop` (ensembler.py:20-187: dense
[Q, 256, 256, 32] mask volumes, a dense soft IoU, ME.to_sparse of every volume) and `panoptic_inference` (helper.py:91-303:
a Python loop over the kept queries with .item() syncs) — the latter where it is used, in both Net modules, which import
it by name.  They return the reference's structures, computed on the sparse rows of predict.py's stages and the dense
emits of csrc/panoptic.cu; inputs outside what the kernels cover (CPU tensors, batch size != 1, more than 8 subnets or 64
classes, rows outside the requested box) go to the saved originals (`_pasco_b200_orig_*`).

The evaluation hook (install(evaluate=True)) replaces `Net.evaluate_all` (net_panoptic_sparse.py:650-765, and the
KITTI-360 Net's) — run in every training and validation step and for every test entry — whose host work copies the
dense volumes with .cpu().numpy(), takes np.unique over 2.1 M uint64 keys and loops in Python per matched segment.  It
runs the dense evaluation passes of csrc/metrics.cu over the volumes it is given (class planes, panoptic ids, voxel
confidences) and finishes the tables with metrics.py's host code into the reference's own PQStat, SSCMetrics and
UncertaintyMetrics objects, with their value types; the ECE is torchmetrics 1.4's binary_calibration_error.  At most
EVAL_SYNCS host synchronisations per call.  CPU tensors, more than 64 classes or one panoptic item, uncertainty
thresholds other than [0.5], volumes whose shapes disagree and labels or predictions outside [0, K) other than 255 go
to the saved original.

The criterion hook (install(criterion=True)) replaces `SetCriterion.compute_losses` (criterion_sparse.py:239-351) — run
for the main and every aux level of every subnet, each re-matched — and the completion losses both Net modules import
by name (losses.py:69-179).  Targets are sampled as bit rows, the matcher's cost sums read the mask logits once
(csrc/setloss.cu), SciPy's assignment stays on the host at the reference's `[Q, T]` copy, the matched-pair focal / dice
and the voxel↔query semantic logits run forward and backward on the kernels, and every Lovász-softmax sorts all classes
in one batched sort.  At most CRITERION_SYNCS host synchronisations per level and per completion-loss call; host
inputs such as the reference's class weights move through pinned memory.  CPU tensors, batch size != 1, a matcher other
than the reference's HungarianMatcher, more than 64 classes or 128 kept queries, no labelled row, and coordinates or
labels outside the label volume go to the saved originals; so do the completion losses' CPU tensors, more than 64
classes, labels beyond the volume, a pair without a present class and (KITTI-360) a pair without a row in bounds.

    import pasco_b200.hooks; pasco_b200.hooks.install()        # after `pasco` is importable, before building Net
    pasco_b200.hooks.install(postprocess=True)                 # the attention and the post-processing
    pasco_b200.hooks.install(postprocess=True, evaluate=True)  # ... and the evaluation
    PASCO_B200_HOOKS=1 python scripts/train.py ...              # compat/MinkowskiEngine calls install() lazily
    PASCO_B200_HOOKS=attention,postprocess,evaluate python scripts/eval.py ...
    PASCO_B200_HOOKS=attention,postprocess,evaluate,criterion python scripts/train.py ...
    PASCO_B200_HOOKS=attention,postprocess,evaluate,criterion,trunk python scripts/train.py ...

The trunk hook (install(trunk=True)) replaces three pieces of the reference's own trunk that run on every training step
and test scene: `CylinderFeat.forward` (unet3d_sparse_v2.py:53-86: torch.unique(dim=0) over all points, a lexicographic
row sort) groups the points with ops.voxel_group (a hash dedup, then a sort of the unique keys only); `Augmenter.merge`
(augmenter.py:13-27: a dense fp32 [M, f, X, Y, Z] volume, copied by torch.cat and scanned by ME.to_sparse, forward and
backward) runs as ops.mimo_merge on the rows; `UNet3DV2.dense_bottleneck` (unet3d_sparse_v2.py:182-214: 11 cuDNN Conv3d
+ BatchNorm3d) runs the reference's SPCDense3Dv2 as box-kernel sparse convolutions over the full stride-8 grid, the
same implementation PascoNet.dense_bottleneck uses (net3d.bottleneck_on_grid).  Grouping and merge are exact; the
bottleneck matches cuDNN's fp32 result within the convolutions' tolerance.  At most TRUNK_SYNCS host synchronisations
per hooked call.  fea_compre, more than 8 subnets, batch size != 1, a dense3d other than (SPCDense3Dv2, Dropout3d), a
Dropout3d with p > 0 in training, coordinates outside [-32768, 32767] and CPU tensors go to the saved originals.

The decoder hook (install(decoder=True)) replaces the glue between the decoder's convolutions, run at every scale and for
every subnet: `DecoderBlock.forward` (decoder_v3.py:148-172) runs `resize` through net3d.resize_rows, the function
PascoNet's decoder stages call (no (C+3)-channel concatenation, the C feature channels on the tensor-core GEMM);
`predict_completion_sem_logit` (:319-394) makes one pasco_completion_rows pass for the argmax, keep masks, cap weights and
counts, read on the host once, and its training cap draws torch.multinomial's Exp(1) variates itself and keeps the k
largest w / q with pasco_topk_mask instead of a full sort (the same rows unless the threshold value occurs twice, the
same generator state); `forward` (:453-511) prunes x and the M logits once per scale; `predict_panop` (:396-451) crops
every subnet and scale with one pasco_panop_crop mask and one compaction, and builds the padded batches and keep_pad
with pasco_mimo_batch on the device, then calls the reference's own transformer_predictor with the original's inputs.
The log lines keep their text.  At most DECODER_SYNCS host synchronisations of the hooks' own per call.  CPU tensors,
more than 8 subnets or 64 classes, logits other than fp32, a resize other than (BatchNorm(C+3), 1x1 convolution), C not
a multiple of 64 in training, a process with an active dropout, bounds that are not 3 integers and logits on another
coordinate map than x go to the saved originals.

The transformer hook (install(transformer=True)) replaces the transformer's dense glue: `PositionEmbeddingSineSparse.forward`
(position_encoding.py:90-135) runs on ops.sine_pos (csrc/posenc.cu, bit for bit) and `TransformerPredictorV2.pred_heads`
(transformer_predictor_v2.py:291-303) on net3d.mask_head (the einsum on ops.linear), both functions PascoNet's
MaskTransformer calls.  With the attention hook, the forward builds voxel_feat and every level's key / value input with
net3d.proj_plus_pos (no [B, P_s, hidden] position tensor; the cross-attention gets pos=None) and each item's outputs
with one compaction and one gather per level.  At most TRANSFORMER_SYNCS host synchronisations of its own per forward.
CPU tensors, normalize=False, a scale other than 2π, odd n or n > 256, float coordinates and a hidden size other than
3n go to the saved originals.
"""
from __future__ import annotations

import collections
import importlib
import math
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

from . import me as ME
from . import metrics, ops, predict


def _transformer_forward(self, xs, sem_logits, min_Cs, max_Cs, keep_pad):
    """transformer_predictor_v2.py:111-218 with the attention masks built on the device as bit rows
    (ops.attention_mask_bits): the reference's own submodules, outputs and padding semantics — padded rows of a MIMO
    batch take part in attention — without its [B·heads, Q, P] bool mask and the int64 row sum of line 164.
    xs[scale] = (F [B, P_s, C], C [B, P_s, 4]) with B = n_infers.  With the transformer group installed too (and a
    pe_layer it covers), the projections add the position encoding into their own rows (net3d.proj_plus_pos: no
    [B, P_s, hidden] position tensor, pos=None to the cross-attention) and each item's outputs are gathered rows
    (_item_outputs)."""
    F1, C1 = xs[1]
    if not F1.is_cuda:
        return self._pasco_b200_orig_forward(xs, sem_logits, min_Cs, max_Cs, keep_pad)
    bs = sem_logits[0].shape[0]
    assert self.n_infers == bs, "batch size should be equal to number of inference"
    glue = _transformer_glue(self, xs)
    output = self.query_feat.weight.reshape(bs, -1, self.hidden_dim)
    query_embed = self.query_embed.weight.reshape(bs, -1, self.hidden_dim)
    if glue:
        pos = [None] * len(self.src_scales)
        voxel_feat = _proj_plus_pos(self.mask_feat_proj, F1, C1, self.pe_layer.num_pos_feats)
    else:
        pos = [self.pe_layer(xs[s][1].reshape(-1, 4)[:, 1:]).reshape(bs, -1, self.hidden_dim) for s in self.src_scales]
        voxel_feat = self.mask_feat_proj(F1) + pos[-1]
    cls, msk = self.pred_heads(output, voxel_feat)
    classes, masks = [cls], [msk]
    voxels = [_voxel_map(c) for c in C1]
    for i, s in enumerate(self.src_scales):
        src_F, src_C = xs[s]
        if glue:
            src_F = _proj_plus_pos(self.input_projs[i], src_F, src_C, self.pe_layer.num_pos_feats)
        else:
            src_F = self.input_projs[i](src_F)
        bits = torch.stack([_mask_bits(voxels[b], masks[-1][b], src_C[b], s) for b in range(bs)])
        output = self.transformer_cross_attention_layers[i](output, src_F, attn_mask=bits, pos=pos[i],
                                                            query_pos=query_embed)
        output = self.transformer_self_attention_layers[i](output, attn_mask=None, padding_mask=None,
                                                           query_pos=query_embed)
        output = self.transformer_ffn_layers[i](output)
        cls, msk = self.pred_heads(output, voxel_feat)
        classes.append(cls)
        masks.append(msk)
    if glue:
        return _item_outputs(self, classes, masks, C1, keep_pad)
    preds = []
    for b in range(bs):
        keep = keep_pad[b]
        item_classes = [c[b].unsqueeze(0) for c in classes]
        item_masks = [ME.SparseTensor(m[b][keep], C1[b][keep]) for m in masks]
        preds.append({"query_logits": item_classes[-1], "voxel_logits": item_masks[-1],
                      "aux_outputs": self.set_aux(item_classes, item_masks)})
    return preds


def _voxel_map(coords: torch.Tensor):
    """One batch item's scale-1 voxels on a coordinate manager of their own: (manager, key, logit row of each unique
    voxel or None).  Padded rows of a MIMO batch share voxel (0,0,0); the first row of a voxel stands for it."""
    C1 = coords.to(torch.int32).clone()
    C1[:, 0] = 0
    mgr = ME.CoordinateManager()
    key1, uidx = mgr.insert_and_map(C1.contiguous())
    return mgr, key1, uidx


def _mask_bits(voxels, logits: torch.Tensor, src_C: torch.Tensor, scale: int) -> torch.Tensor:
    """transformer_predictor_v2.py:220-289 and 164 for one batch item: logits [P1, Q], src_C [P_s, 4] →
    ops.attention_mask_bits' int32 bit rows [Q, 2*ceil(P_s/64)]."""
    mgr, key1, uidx = voxels
    parent_of, key_s = None, key1
    if scale != 1:
        key_s = mgr.stride(key1, scale)
        parent_of = mgr.pool_map(key1, key_s, scale)
    Cs = src_C.to(torch.int32).clone()
    Cs[:, 0] = 0
    return ops.attention_mask_bits(logits.detach(), ops.hash_lookup(mgr._table(key_s), Cs.contiguous()), uidx,
                                   parent_of, mgr.size(key_s))


def _cross_attention_forward(self, q_embed, bb_feat, attn_mask=None, padding_mask=None, pos=None, query_pos=None):
    """blocks.py:73-92 with the attention on xattn.cu, for the bit-row masks [B, Q, words] the hooked
    TransformerPredictorV2.forward passes; any other mask (the reference's bool [B·heads, Q, P]) goes to the original.
    q_embed [B, Q, d]; bb_feat / pos [B, P, d]."""
    if attn_mask is None or attn_mask.dtype != torch.int32 or padding_mask is not None or not bb_feat.is_cuda:
        return self._pasco_b200_orig_forward(q_embed, bb_feat, attn_mask, padding_mask, pos, query_pos)
    q_embed = self.norm(q_embed)
    outs = []
    for b in range(q_embed.shape[0]):
        qb = q_embed[b] if query_pos is None else q_embed[b] + query_pos[b]
        kv = bb_feat[b] if pos is None else bb_feat[b] + pos[b]
        outs.append(ops.cross_attention(self.multihead_attn, qb, kv, attn_mask[b]))
    return q_embed + self.dropout(torch.stack(outs, 0))


# ------------------------------------------------------------------------------------------------
# transformer glue: PositionEmbeddingSineSparse.forward (position_encoding.py:90-135) on ops.sine_pos,
# TransformerPredictorV2.pred_heads (transformer_predictor_v2.py:291-303) on net3d.mask_head, and with the attention
# group the projections and per-item outputs of _transformer_forward
# ------------------------------------------------------------------------------------------------
TRANSFORMER_SYNCS = 1   # host synchronisations of the group's own code in one hooked forward, at most: the kept row
                        # counts of every item (_item_outputs)


def _pe_covered(pe) -> bool:
    """The encodings ops.sine_pos computes: normalize=True with the default scale 2π, n even and at most 256."""
    n = getattr(pe, "num_pos_feats", None)
    return (getattr(pe, "normalize", False) is True and getattr(pe, "scale", None) == 2 * math.pi
            and isinstance(n, int) and n % 2 == 0 and 2 <= n <= 256)


def _transformer_glue(self, xs) -> bool:
    """Whether _transformer_forward runs the group's glue: the transformer and attention groups installed, a pe_layer
    that _pe_covered covers with hidden_dim = 3n, and integer coordinates at every source scale."""
    pe = self.pe_layer
    return ("transformer" in _installed and "attention" in _installed and _pe_covered(pe)
            and self.hidden_dim == 3 * pe.num_pos_feats
            and all(xs[s][1].dtype in (torch.int32, torch.int64) for s in self.src_scales))


def _pe_forward(self, coords):
    """position_encoding.py:90-135 on ops.sine_pos, the same values bit for bit.  CPU tensors, float coordinates, rows
    other than [N, 3] and encodings _pe_covered does not cover go to the saved original."""
    if not (_pe_covered(self) and torch.is_tensor(coords) and coords.is_cuda and coords.dim() == 2
            and coords.shape[1] == 3 and coords.dtype in (torch.int32, torch.int64)):
        return self._pasco_b200_orig_forward(coords)
    return ops.sine_pos(coords, self.num_pos_feats, temperature=self.temperature)


def _pred_heads(self, output, mask_features):
    """transformer_predictor_v2.py:291-303 as net3d.mask_head: class logits from the module's own layers, the mask
    einsum on ops.linear.  CPU tensors and inputs other than fp32 [B, Q, d] / [B, P, d] go to the saved original."""
    from .net3d import mask_head
    if not (output.is_cuda and mask_features.is_cuda and output.dim() == 3 and mask_features.dim() == 3
            and output.dtype == torch.float32 and mask_features.dtype == torch.float32
            and output.shape[0] == mask_features.shape[0] and output.shape[2] == mask_features.shape[2]):
        return self._pasco_b200_orig_pred_heads(output, mask_features)
    return mask_head(self, output, mask_features)


def _proj_plus_pos(linear, F_: torch.Tensor, C: torch.Tensor, n: int) -> torch.Tensor:
    """net3d.proj_plus_pos over a padded batch: F [B, P, Cin], C [B, P, 4] → [B, P, 3n]."""
    from .net3d import proj_plus_pos
    B, P = F_.shape[0], F_.shape[1]
    return proj_plus_pos(linear, F_.reshape(B * P, -1), C.reshape(B * P, C.shape[-1]), n).reshape(B, P, -1)


def _item_outputs(self, classes, masks, C1, keep_pad):
    """transformer_predictor_v2.py:190-216 without its boolean indexings, hash inserts and syncs per level: one
    compaction of keep_pad[b] per item (every item's kept count read in one synchronisation) and, per level, one
    gather of the logit rows and one of the coordinates, registered on a coordinate manager of the level's own.  Each
    level's .C is thus a tensor of its own: SetCriterion.compute_losses shifts pred_mask_C by min_C in place.  keep_pad
    selects one subnet's rows of a coordinate map, which are unique, so the maps are registered without a dedup."""
    kp = keep_pad if torch.is_tensor(keep_pad) else torch.stack(list(keep_pad))
    counts = kp.sum(1).tolist()                                                              # the one sync
    preds = []
    for b, n_keep in enumerate(counts):
        kept, _, _ = ops.compact(kp[b], int(n_keep))
        Cb = C1[b].to(torch.int32).contiguous()
        item_masks = []
        for m in masks:
            mgr = ME.CoordinateManager()
            key = mgr._register(ops.gather_coords(Cb, kept), 1)
            item_masks.append(ME.SparseTensor(ops.GatherRows.apply(m[b], kept), coordinate_map_key=key,
                                              coordinate_manager=mgr))
        item_classes = [c[b].unsqueeze(0) for c in classes]
        preds.append({"query_logits": item_classes[-1], "voxel_logits": item_masks[-1],
                      "aux_outputs": self.set_aux(item_classes, item_masks)})
    return preds


# ------------------------------------------------------------------------------------------------
# post-processing: Ensembler.ensemble_sem_compl / ensemble_panop (ensembler.py:20-187) and panoptic_inference
# (helper.py:91-303) on the row-form kernels of csrc/panoptic.cu (predict.py's stages)
# ------------------------------------------------------------------------------------------------
def _saved(module: str, name: str):
    """The original of `module`'s module-level `name` as install() saved it (`_pasco_b200_orig_<name>` on the module),
    read when called."""
    return lambda *args: getattr(importlib.import_module(module), "_pasco_b200_orig_" + name)(*args)


_orig_panoptic_inference = _saved("pasco.models.helper", "panoptic_inference")   # the Net modules import the same one


def _rows_at(lin: torch.Tensor, size=predict.SCENE) -> torch.Tensor:
    """Ascending cells → int32 [n, 4] (0, x, y, z) rows, ME.to_sparse's coordinates."""
    lin = lin.long()
    Y, Z = int(size[1]), int(size[2])
    return torch.stack([torch.zeros_like(lin), lin // (Y * Z), (lin // Z) % Y, lin % Z], 1).to(torch.int32).contiguous()


def _ensemble_sem_compl(self, sem_logits_at_scales, Ts):
    """ensembler.py:159-187: the M + 1 dense class distributions [K, 256, 256, 32] from the softmax rows of every subnet.
    The ensemble's occupancy gate is kept on the instance for the ensemble_panop call that follows."""
    sems = sem_logits_at_scales[1]
    self._pasco_b200_sem_state = None
    if len(sems) > 8 or sems[0].F.shape[1] > 64 or not all(s.F.is_cuda for s in sems):
        return self._pasco_b200_orig_ensemble_sem_compl(sem_logits_at_scales, Ts)
    rows = predict.semantic_rows([(s.F, s.C) for s in sems], Ts)
    cells = predict.SCENE[0] * predict.SCENE[1] * predict.SCENE[2]
    gate = torch.empty(cells, dtype=torch.uint8, device=rows[0][0].device)
    subs, ens = ops.sem_dense([p for p, _, _ in rows], [c for _, _, c in rows], cells, gate=gate)
    out = [v.view(-1, *predict.SCENE) for v in subs + [ens]]
    self._pasco_b200_sem_state = (out[-1], gate)
    return out


def _ensemble_panop(self, panop_predictions, ensemble_sem_prob_denses, scene_size, Ts, iou_threshold=0.2,
                    measure_time=False):
    """ensembler.py:20-131 on rows: {"sem_probs", "voxel_probs", "query_probs"} per subnet and for the ensemble, the
    voxel probabilities on a fresh coordinate manager in ME.to_sparse order (ascending cell of the 256 x 256 x 32 grid,
    all-zero rows dropped).  measure_time: "ensemble_time" covers the matching and the merge, as the reference times it
    (ensembler.py:69-113), not the per-subnet warps before it."""
    ql = panop_predictions[0]["query_logits"]
    ens_vol = ensemble_sem_prob_denses[-1]
    if (len(panop_predictions) > 8 or ql.shape[0] != 1 or not ql.is_cuda or not ens_vol.is_cuda
            or ens_vol.shape[0] > 64 or tuple(ens_vol.shape[1:]) != predict.SCENE
            or not all(p["voxel_logits"].F.is_cuda for p in panop_predictions)):
        return self._pasco_b200_orig_ensemble_panop(panop_predictions, ensemble_sem_prob_denses, scene_size, Ts,
                                                    iou_threshold=iou_threshold, measure_time=measure_time)
    state = getattr(self, "_pasco_b200_sem_state", None)
    self._pasco_b200_sem_state = None                 # used once: do not keep the volume alive past this scene
    gate = state[1] if state is not None and state[0] is ens_vol else ops.class_gate(ens_vol)
    preds = [{"voxel_logits": (p["voxel_logits"].F, p["voxel_logits"].C), "query_logits": p["query_logits"]}
             for p in panop_predictions]
    masks, qprobs = predict.mask_warps(preds, Ts)
    if measure_time:
        torch.cuda.synchronize()
        t0 = time.time()
    rows, qprobs = predict.mask_rows(masks, qprobs, gate, iou_threshold=iou_threshold)
    if measure_time:
        torch.cuda.synchronize()
        ensemble_time = time.time() - t0
    out = []
    for (prob, lin), qp, sem_dense in zip(rows, qprobs, ensemble_sem_prob_denses):
        coords = _rows_at(lin)
        sem = ops.from_dense_raw(sem_dense.detach().float().unsqueeze(0).contiguous(), coords, (0, 0, 0), (1, 1, 1))
        entry = {"sem_probs": ME.SparseTensor(sem, coords), "voxel_probs": ME.SparseTensor(prob, coords),
                 "query_probs": qp}
        if measure_time:
            entry["ensemble_time"] = ensemble_time
        out.append(entry)
    return out


def _squeezed(t: torch.Tensor) -> torch.Tensor:
    """helper.py:264-281: to_dense_tensor's [C, X, Y, Z] volume with C = 1 for the per-voxel outputs, then .squeeze()."""
    return t.unsqueeze(0).squeeze()


def _panoptic_inference(voxel_output, query_output, overlap_threshold, object_mask_threshold, thing_ids, min_C,
                        scene_size, input_query_logit=True, input_voxel_logit=False, vox_occ_threshold=0.3):
    """helper.py:91-303 for batch size 1 on pasco_panoptic_pass1 / segments / pass2 / dense: the reference's dict with its
    shapes and dtypes.  Two host synchronisations (the segment records, the box check), plus one for each of min_C and
    scene_size given as device tensors (Net.step's call) — whatever the query count."""
    args = (voxel_output, query_output, overlap_threshold, object_mask_threshold, thing_ids, min_C, scene_size,
            input_query_logit, input_voxel_logit, vox_occ_threshold)
    F_ = voxel_output.F
    Q, K1 = query_output.shape[1], query_output.shape[-1]
    if (query_output.shape[0] != 1 or not (F_.is_cuda and query_output.is_cuda) or not 2 <= K1 <= 65
            or not 1 <= Q <= 8192 or F_.shape[1] != Q):
        return _orig_panoptic_inference(*args)
    voxel_probs = ME.MinkowskiSigmoid()(voxel_output) if input_voxel_logit else voxel_output
    qp = F.softmax(query_output[0], dim=-1) if input_query_logit else query_output[0]
    coords = voxel_probs.C.to(torch.int32).contiguous()
    min_c = [int(v) for v in torch.as_tensor(min_C).reshape(-1).tolist()]
    size = [int(v) for v in (scene_size.tolist() if torch.is_tensor(scene_size) else scene_size)]
    pan_rows, records, vol = ops.panoptic_dense(voxel_probs.F.detach().float(), coords, qp, overlap_threshold,
                                                object_mask_threshold, thing_ids, min_c, size, vox_occ_threshold)
    if vol is None:                                    # a row outside the box: the reference's own indexing decides
        return _orig_panoptic_inference(*args)
    return {
        "vox_all_mask_probs_denses": [vol["all_mask_probs"].squeeze()],
        "panoptic_seg_denses": _squeezed(vol["panoptic"]).unsqueeze(0),
        "semantic_seg_denses": _squeezed(vol["semantic"]).unsqueeze(0),
        "ins_uncertainty_denses": _squeezed(vol["ins_uncertainty"]).unsqueeze(0),
        "vox_confidence_denses": _squeezed(vol["confidence"]).unsqueeze(0),
        "vox_uncertainty_denses": _squeezed(vol["vox_uncertainty"]).unsqueeze(0),
        "panoptic_seg_sparses": [pan_rows],
        "segments_infos": [predict._segments(records, qp)],
    }


# ------------------------------------------------------------------------------------------------
# evaluation: Net.evaluate_all (net_panoptic_sparse.py:650-765) on the dense forms of csrc/metrics.cu, finished by
# metrics.py's host code into the reference's own metric objects
# ------------------------------------------------------------------------------------------------
EVAL_SYNCS = 3          # host synchronisations of a hooked evaluate_all call, at most (see _evaluate)


def _ref_iou(inter: int, union: int):
    """The reference's pair IoU: np.int64 intersection / a 0-d torch area, i.e. Tensor.__rdiv__ = reciprocal() * other,
    in float32."""
    return (np.float32(1.0) / np.float32(union)) * np.float32(inter)


class _SeededCats(dict):
    """metrics.finish_pq's category mapping over a PQStat: a category first touched starts from the PQStat's current
    fields (device iou sums as their host values), so the float32 sums continue in the reference's order."""

    def __init__(self, pq_stat, prev):
        super().__init__()
        self.pq, self.prev = pq_stat, prev

    def __missing__(self, c):
        cat = metrics._Cat()
        old = self.pq.pq_per_cat.get(c)
        if old is not None:
            cat.all_n, cat.tp, cat.fp, cat.fn = old.all_n, old.tp, old.fp, old.fn
            cat.all_iou = self.prev.get((c, "all_iou"), old.all_iou)
            cat.iou = self.prev.get((c, "iou"), old.iou)
        self[c] = cat
        return cat


def _host_copy(t: torch.Tensor) -> torch.Tensor:
    """A pinned host copy, enqueued on the stream: complete at the call's next synchronisation."""
    h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    h.copy_(t, non_blocking=True)
    return h


def _evaluate(net, ssc_confidence, i_infer, sem_prob, panop_out, semantic_label, mask_labels, ssc_metrics, pq_stat,
              compute_uncertainty, inference_time):
    """evaluate_all on the device, or None where the saved original decides (the caller then runs it; nothing has been
    updated).  Host synchronisations: one to read mask_labels["labels"] when it is a device tensor, one for every
    counting table and the returned volumes, and with compute_uncertainty one for the voxel calibration table — at most
    EVAL_SYNCS, whatever the query, segment or cell counts."""
    pan_all = panop_out["panoptic_seg_denses"]
    if not (torch.is_tensor(sem_prob) and sem_prob.is_cuda and sem_prob.dtype == torch.float32 and sem_prob.dim() == 4
            and torch.is_tensor(pan_all) and len(pan_all) == 1 and torch.is_tensor(semantic_label)):
        return None
    dev, K, size = sem_prob.device, sem_prob.shape[0], tuple(sem_prob.shape[1:])
    cells = sem_prob[0].numel()
    ml = mask_labels[0]
    masks = ml["masks"]
    thresholds = list(getattr(net, "uncertainty_thresholds", [0.5]))
    pan = pan_all[0]
    if (K > 64 or K != ssc_metrics.n_classes or min(size) < 2 or tuple(semantic_label.shape) != (1,) + size
            or semantic_label.device != dev or semantic_label.dtype.is_floating_point or semantic_label.dtype == torch.bool
            or pan.device != dev or pan.dtype != torch.int32 or tuple(pan.shape) != size
            or not (torch.is_tensor(masks) and masks.device == dev and masks.dim() == 4 and tuple(masks.shape[1:]) == size)
            or not hasattr(pq_stat, "pq_per_cat")):
        return None
    if compute_uncertainty:
        vconf = panop_out["vox_confidence_denses"][0]
        if (thresholds != [0.5] or not torch.is_tensor(ssc_confidence) or ssc_confidence.device != dev
                or ssc_confidence.dtype != torch.float32 or ssc_confidence.numel() != cells
                or not torch.is_tensor(vconf) or vconf.device != dev or vconf.dtype != torch.float32
                or tuple(vconf.shape) != size):
            return None
    # the PQStat's float32 iou sums so far: device tensors are read with the tables below
    prev_t = []
    for c, s in pq_stat.pq_per_cat.items():
        for f in ("all_iou", "iou"):
            v = getattr(s, f)
            if torch.is_tensor(v):
                if not (v.device == dev and v.dtype == torch.float32 and v.numel() == 1):
                    return None
                prev_t.append(((c, f), v.reshape(1)))

    # ground truth (convert_mask_label_to_panoptic_output's walk on the host, the mask stack on the device)
    labels = ml["labels"]
    labels = labels.reshape(-1).tolist() if torch.is_tensor(labels) else list(labels)      # sync 1 for device labels
    if any(int(v) != v or not (0 <= v < K or v == 255) for v in labels) or len(labels) != masks.shape[0]:
        return None
    labels = [int(v) for v in labels]
    seg_of, segs = metrics.gt_walk(labels, net.thing_ids)
    n, G = len(labels), len(segs)
    label = semantic_label.reshape(-1)
    if label.dtype != torch.uint8:                     # anything outside [0, K) other than 255 reads as K: the fallback
        label = torch.where(((label >= 0) & (label < K)) | (label == 255), label, K).to(torch.uint8)
    label = label.contiguous()
    m8 = masks.reshape(n, cells)
    m8 = m8.contiguous().view(torch.uint8) if m8.dtype == torch.bool else (m8 != 0).contiguous().view(torch.uint8)
    seg = torch.tensor(seg_of, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
    gt_id, counts = ops.eval_gt(m8, seg, label, G, K)
    gt_host = _host_copy(ops.eval_gt_volume(gt_id))

    # the entry: (gt id, pred id) pairs, and the SSC pass over the class planes
    seg_infos = panop_out["segments_infos"][0]
    ids = [int(s["id"]) for s in seg_infos]
    S = max(ids + [0])
    t_pairs = (G + 1) * (S + 1) + S + 1
    o_ssc = t_pairs + t_pairs % 2
    o_sum = K * K + 65 + (K * K + 65) % 2
    tab = torch.zeros(o_ssc + o_sum + 68, dtype=torch.int32, device=dev)
    ops.eval_pairs_dense(pan.contiguous(), gt_id, label, G, S, tab[:t_pairs])
    pred = ops.eval_ssc_planes(sem_prob.reshape(K, cells).contiguous(), label,
                               ssc_confidence.reshape(-1).contiguous() if compute_uncertainty else None, tab[o_ssc:])
    pred_host = _host_copy(pred)
    parts = [tab, counts] + ([torch.cat([v for _, v in prev_t]).view(torch.int32)] if prev_t else [])
    host = torch.cat(parts).cpu()                                                            # sync 2
    h = host.numpy()
    t, counts_h = h[:tab.numel()], h[tab.numel():tab.numel() + counts.numel()]
    prev = {k: np.float32(v) for (k, _), v in zip(prev_t, h[tab.numel() + counts.numel():].view(np.float32))}
    mask_sum, id_area, hist = counts_h[:n], counts_h[n:n + G + 1], counts_h[n + G + 1:]
    pairs = t[:(G + 1) * (S + 1)].reshape(G + 1, S + 1)
    pred_area = t[(G + 1) * (S + 1):t_pairs]
    conf = t[o_ssc:o_ssc + K * K].reshape(K, K).astype(np.int64)
    cal = t[o_ssc + K * K:o_ssc + K * K + 64].reshape(2, 2, 16).astype(np.float64)
    bad = int(t[o_ssc + K * K + 64])
    sums = host[o_ssc + o_sum:o_ssc + o_sum + 68].view(torch.float64).numpy()                # 8-byte aligned
    present = set(np.nonzero(pred_area)[0].tolist()) - {0}
    if hist[K] or bad or pred_area[0] or not present <= set(ids):
        return None                  # labels or confidences outside the covered range, or ids without a segment

    # panoptic quality into the PQStat, in the reference's order and value types
    gt_area = {sid: int(mask_sum[i]) for sid, _, _, i in segs}
    gt_segs = [(sid, c) for sid, c, _, _ in segs if id_area[sid] > 0]
    pred_kept = [s for s in seg_infos if int(s["id"]) in present]
    pred_segs = [(int(s["id"]), int(s["category_id"])) for s in pred_kept]
    cats = _SeededCats(pq_stat, prev)
    _, _, unc = metrics.finish_pq(cats, pairs, pred_area, gt_area, gt_segs, pred_segs, net.thing_ids, iou_of=_ref_iou)

    vox = None
    if compute_uncertainty:
        match = np.zeros(S + 1, np.int32)
        for p, g in unc.items():
            match[p] = g
        vt = torch.zeros(66, dtype=torch.int32, device=dev)
        ops.eval_vox_dense(pan.contiguous(), vconf.contiguous(), gt_id,
                           torch.from_numpy(match).pin_memory().to(dev, non_blocking=True), vt)
        vh = vt.cpu()                                                                        # sync 3
        if int(vh[64]):
            return None
        vox = vh[:32].numpy().reshape(2, 16), vh[32:64].view(torch.float64).numpy()

    # ---- nothing has been updated so far; from here on the call writes the reference's objects
    tensor_fields = [(c, f, getattr(cat, f)) for c, cat in cats.items() for f in ("all_iou", "iou")
                     if isinstance(getattr(cat, f), np.float32)]
    vals = torch.tensor([float(v) for _, _, v in tensor_fields], dtype=torch.float32).pin_memory().to(
        dev, non_blocking=True)
    j = {(c, f): i for i, (c, f, _) in enumerate(tensor_fields)}
    for c, cat in cats.items():
        st = pq_stat[c]
        st.tp, st.fp, st.fn, st.all_n = cat.tp, cat.fp, cat.fn, cat.all_n
        for f in ("all_iou", "iou"):
            if (c, f) in j:
                setattr(st, f, vals[j[c, f]])
    for s in pred_kept:                                # pq_compute_single_core records each kept segment's area
        s["area"] = np.int64(pred_area[int(s["id"])])

    tp, fp, fn = int(conf[1:, 1:].sum()), int(conf[0, 1:].sum()), int(conf[1:, 0].sum())
    diag = np.diag(conf)
    ssc_metrics.completion_tp += tp
    ssc_metrics.completion_fp += fp
    ssc_metrics.completion_fn += fn
    ssc_metrics.tps += diag
    ssc_metrics.fps += conf.sum(0) - diag
    ssc_metrics.fns += conf.sum(1) - diag

    if compute_uncertainty:
        ssc_metrics.empty_nll += float(sums[32])
        ssc_metrics.nonempty_nll += float(sums[33])
        ssc_metrics.n_empty_voxels += int(cal[0, 0].sum())
        ssc_metrics.n_nonempty_voxels += int(cal[1, 0].sum())
        ssc_metrics.empty_ece += metrics.ece_from_bins(cal[0, 0], sums[:16], cal[0, 1])
        ssc_metrics.nonempty_ece += metrics.ece_from_bins(cal[1, 0], sums[16:32], cal[1, 1])
        ssc_metrics.ece_count += 1
        ssc_metrics.inference_time += inference_time

        um = net.uncertainty_metrics_by_thresholds[0.5][i_infer]
        gcat = dict(gt_segs)
        for s in pred_kept:                            # compute_ece_panop (metrics.py:98-165)
            g = unc.get(int(s["id"]))
            um.ins_confs.append(s["confidence"])
            um.ins_all_class_probs.append(s["all_class_probs"])
            um.ins_sem_labels.append(net.n_classes if g is None else gcat[g])
            um.ins_correct.append(g is not None and gcat[g] == s["category_id"])
        vc, vs = vox
        um.mask_ece += metrics.ece_from_bins(vc[0], vs, vc[1]) if vc[0].sum() else 0
        um.mask_auprc += 0
        um.mask_auroc += 0
        um.mask_fpr95 += 0
        um.count += 1

    areas = counts[:n].to(torch.int64)
    gt_segments_info = [{"id": sid, "isthing": isthing, "category_id": c, "area": areas[i]}
                        for sid, c, isthing, i in segs if id_area[sid] > 0]
    return gt_host.numpy().reshape(size), gt_segments_info, pred_host.numpy().reshape((1,) + size)


def _evaluate_all(self, ssc_confidence, i_infer, sem_prob, panop_out, semantic_label, mask_labels, ssc_metrics,
                  pq_stat, uncertainty_metrics, compute_uncertainty=False, inference_time=0.0):
    """net_panoptic_sparse.py:650-695 on the dense evaluation passes: the reference's metric objects updated in place,
    its (gt_panoptic_seg, gt_segments_info, ssc_pred) returned."""
    with torch.no_grad():
        out = _evaluate(self, ssc_confidence, i_infer, sem_prob, panop_out, semantic_label, mask_labels, ssc_metrics,
                        pq_stat, compute_uncertainty, inference_time)
    if out is None:
        return self._pasco_b200_orig_evaluate_all(
            ssc_confidence=ssc_confidence, i_infer=i_infer, sem_prob=sem_prob, panop_out=panop_out,
            semantic_label=semantic_label, mask_labels=mask_labels, ssc_metrics=ssc_metrics, pq_stat=pq_stat,
            uncertainty_metrics=uncertainty_metrics, compute_uncertainty=compute_uncertainty,
            inference_time=inference_time)
    return out


def _evaluate_all_kitti360(self, ssc_confidence, i_infer, sem_prob, panop_out, semantic_label, mask_labels,
                           ssc_metrics, pq_stat, uncertainty_metrics, compute_uncertainty=False):
    """net_panoptic_sparse_kitti360.py:485-518: the same, without inference_time."""
    with torch.no_grad():
        out = _evaluate(self, ssc_confidence, i_infer, sem_prob, panop_out, semantic_label, mask_labels, ssc_metrics,
                        pq_stat, compute_uncertainty, 0.0)
    if out is None:
        return self._pasco_b200_orig_evaluate_all(
            ssc_confidence=ssc_confidence, i_infer=i_infer, sem_prob=sem_prob, panop_out=panop_out,
            semantic_label=semantic_label, mask_labels=mask_labels, ssc_metrics=ssc_metrics, pq_stat=pq_stat,
            uncertainty_metrics=uncertainty_metrics, compute_uncertainty=compute_uncertainty)
    return out


# ------------------------------------------------------------------------------------------------
# training criterion: SetCriterion.compute_losses (criterion_sparse.py:239-351) and the completion losses
# (losses.py:69-179) on csrc/setloss.cu
# ------------------------------------------------------------------------------------------------
CRITERION_SYNCS = 1     # host synchronisations of one hooked compute_losses level or completion-loss call, at most


_pinned_to = ops.pinned_to
_on = ops.on_device


def _criterion_level(crit, outputs, targets, semantic_label, unknown_mask_dense, i_infer, min_C):
    """compute_losses for batch size 1 → (loss_label_agg, loss_mask_agg), or None where the saved original decides.
    The device work is criterion.DeviceCriterion's for one level with its ssc term: one host synchronisation for the
    cost matrix, the sampling counters and the kept-query count, at the reference's own crossing before
    linear_sum_assignment.  What stays here is the reference's: its objects, `loss_labels` and `CE_ssc_loss`."""
    from pasco.loss.losses import CE_ssc_loss
    from pasco.loss.matcher_sparse import HungarianMatcher
    from .criterion import MAX_CLASSES, DeviceCriterion
    vl, ql = outputs["voxel_logits"], outputs["query_logits"]
    if len(targets) != 1 or type(crit.matcher) is not HungarianMatcher or min_C is None:
        return None
    F_, labels, masks = vl.F, targets[0]["labels"], targets[0]["masks"]
    dev = F_.device
    if not (F_.is_cuda and ql.is_cuda and torch.is_tensor(masks) and masks.device == dev and masks.dim() == 4):
        return None
    K1 = ql.shape[-1]
    K, Q, size = K1 - 1, F_.shape[1], tuple(masks.shape[1:])
    if not (1 <= K <= MAX_CLASSES and Q == ql.shape[-2] and Q <= 4096 and tuple(unknown_mask_dense.shape) == (1,) + size
            and tuple(semantic_label.shape) == (1,) + size and unknown_mask_dense.device == dev
            and semantic_label.device == dev and F_.dtype == torch.float32):
        return None
    pred_logit = ql[0]
    dc = DeviceCriterion(dev)
    dc.add_subnet(vl.C, min_C, masks, unknown_mask_dense[0], semantic_label[0], labels, crit.class_weights[i_infer], K,
                  [(F_, pred_logit, True)])
    if not dc.read(crit.matcher):
        return None                 # rows outside the volume, labels outside [0, K), no labelled row, > 128 kept
    dc.run()
    lv, sub = dc.levels[0], dc.subnets[0]
    qi_d, tj_d, class_weight = lv["qi"], lv["tj"], sub["cw"]

    loss_label_agg = {"loss_ce": 0}
    loss_mask_agg = {"loss_mask": 0, "loss_dice": 0, "ssc_ce_loss": 0, "ssc_lovasz_loss": 0}
    # loss_labels (criterion_sparse.py:56-81) itself, given the assignment as device indices
    loss_label = crit.loss_labels({"query_logits": pred_logit}, {"labels": sub["labels"]}, (qi_d.long(), tj_d.long()),
                                  class_weight)
    # loss_masks (criterion_sparse.py:83-112) from the per-pair sums over the known rows
    loss_mask, loss_dice = DeviceCriterion.mask_dice(lv, class_weight[sub["ids"][tj_d.long()].long()])
    loss_label_agg["loss_ce"] += (loss_label["loss_ce"] * crit.weight_dict["loss_ce"]).mean()
    loss_mask_agg["loss_mask"] += (loss_mask * crit.weight_dict["loss_mask"]).mean()
    loss_mask_agg["loss_dice"] += (loss_dice * crit.weight_dict["loss_dice"]).mean()

    # compute_ssc_sparse_loss (criterion_sparse.py:180-209)
    ssc_ce_loss, ssc_lovasz_loss = 0, 0
    if lv["ssc_logits"] is not None:
        lab = sub["lab"]
        ssc_ce_loss += CE_ssc_loss(lv["ssc_logits"], torch.where(lab < 0, 0, lab).long(), crit.compl_labelweights)
        if lv["ssc_lovasz"] is not None:
            ssc_lovasz_loss += lv["ssc_lovasz"]
    loss_mask_agg["ssc_ce_loss"] += ssc_ce_loss * crit.weight_dict["ssc_ce"]
    loss_mask_agg["ssc_lovasz_loss"] += ssc_lovasz_loss * crit.weight_dict["ssc_lovasz"]
    return loss_label_agg, loss_mask_agg


def _compute_losses(self, sem_logits_pruned_1_1, outputs, targets, semantic_label, unknown_mask_dense, i_infer,
                    indices=[], min_C=None):  # noqa: B006  (the reference's signature)
    """criterion_sparse.py:239-351 on csrc/setloss.cu: the reference's (loss_label_agg, loss_mask_agg, indices) with
    its keys and value types.  Inputs the kernels do not cover go to the saved original."""
    out = _criterion_level(self, outputs, targets, semantic_label, unknown_mask_dense, i_infer, min_C)
    if out is None:
        return self._pasco_b200_orig_compute_losses(sem_logits_pruned_1_1, outputs, targets, semantic_label,
                                                    unknown_mask_dense, i_infer, indices, min_C)
    return out[0], out[1], indices


def _sem_compl_loss(sem_labels, sem_logits_at_scales, min_Cs, max_Cs, class_frequencies, power, skip_empty):
    """losses.py:124-179 (power 1/3, pairs without a row inside the bounds skipped) and :71-121 (power 1/1.5) →
    (CE, Lovász), or None where the saved original decides.  The device work is criterion.DeviceCriterion's for all
    (scale, subnet) pairs: one host synchronisation for their in-bounds row counts and present classes."""
    from .criterion import MAX_CLASSES, DeviceCriterion, label_weights
    dc = None
    for scale in sem_logits_at_scales:
        sem_logits = sem_logits_at_scales[scale]
        targets = sem_labels["1_{}".format(scale)]
        w = label_weights(class_frequencies["1_{}".format(scale)], power).tolist()
        for i_subnet in range(len(targets)):
            sl, target = sem_logits[i_subnet], targets[i_subnet]
            if not (sl.F.is_cuda and torch.is_tensor(target) and target.device == sl.F.device and target.dim() == 3
                    and sl.F.dtype == torch.float32 and 1 <= sl.F.shape[1] <= MAX_CLASSES):
                return None
            dc = dc or DeviceCriterion(sl.F.device)
            dc.add_pair(sl, target, min_Cs[i_subnet], max_Cs[i_subnet], scale, w)
    if dc is None:
        return None
    if not dc.read(None, skip_empty):
        return None             # labels beyond the volume, no present class, or an empty pair the original decides
    dc.run()
    live = [pr for pr in dc.pairs if pr["n_in"] > 0]
    if len(live) == 0:
        return 0.0, 0.0
    return torch.stack([pr["ce"] for pr in live]).mean(), torch.stack([pr["lovasz"] for pr in live]).mean()


def _compute_sem_compl_loss(sem_labels, sem_logits_at_scales, min_Cs, max_Cs, class_frequencies):
    """losses.py:124-179 with the Lovász-softmax on csrc/setloss.cu."""
    out = _sem_compl_loss(sem_labels, sem_logits_at_scales, min_Cs, max_Cs, class_frequencies, 1 / 3.0, True)
    if out is None:
        return _orig_compl[0](sem_labels, sem_logits_at_scales, min_Cs, max_Cs, class_frequencies)
    return out


def _compute_sem_compl_loss_kitti360(sem_labels, sem_logits_at_scales, min_Cs, max_Cs, class_frequencies):
    """losses.py:71-121 (KITTI-360 label weights) with the Lovász-softmax on csrc/setloss.cu."""
    out = _sem_compl_loss(sem_labels, sem_logits_at_scales, min_Cs, max_Cs, class_frequencies, 1 / 1.5, False)
    if out is None:
        return _orig_compl[1](sem_labels, sem_logits_at_scales, min_Cs, max_Cs, class_frequencies)
    return out


# the Net modules' compute_sem_compl_loss / compute_sem_compl_loss_kitti360 as install() found them
_orig_compl = [_saved("pasco.models.net_panoptic_sparse", "compute_sem_compl_loss"),
               _saved("pasco.models.net_panoptic_sparse_kitti360", "compute_sem_compl_loss_kitti360")]


# ------------------------------------------------------------------------------------------------
# trunk: CylinderFeat.forward (unet3d_sparse_v2.py:53-86), Augmenter.merge (augmenter.py:13-27) and
# UNet3DV2.dense_bottleneck (unet3d_sparse_v2.py:182-214) on csrc/voxel.cu and net3d's grid bottleneck
# ------------------------------------------------------------------------------------------------
TRUNK_SYNCS = 4     # host synchronisations of one hooked trunk call, at most (see each function)


def _cylinder_forward(self, pt_fea, xy_ind):
    """unet3d_sparse_v2.py:53-86 with torch.unique(dim=0) as ops.voxel_group and the scatter-max on
    ops.scatter_max; the point MLP is the reference's own PPmodel.  The randperm is drawn but not applied: the CUDA
    generator ends where the original leaves it, and the max does not depend on the point order (only the rounding of
    the BatchNorm1d batch statistics does).  One host synchronisation (the voxel count)."""
    if self.fea_compre is not None or not (pt_fea[0].is_cuda and xy_ind[0].is_cuda):
        return self._pasco_b200_orig_forward(pt_fea, xy_ind)
    cat_pt_ind = torch.cat([F.pad(xy_ind[b], (1, 0), "constant", value=b) for b in range(len(xy_ind))], dim=0)
    if cat_pt_ind.dtype not in (torch.int32, torch.int64):
        return self._pasco_b200_orig_forward(pt_fea, xy_ind)
    grouped = ops.voxel_group(cat_pt_ind)
    if grouped is None:                                # a coordinate the packed keys cannot hold
        return self._pasco_b200_orig_forward(pt_fea, xy_ind)
    torch.randperm(cat_pt_ind.shape[0], device=pt_fea[0].get_device())
    unq, inv = grouped
    processed = self.PPmodel(torch.cat(pt_fea, dim=0))
    pooled = ops.scatter_max(processed, inv, dim=0, dim_size=unq.shape[0])[0]
    return unq.to(torch.int64), pooled


def _augmenter_merge(self, in_feat):
    """augmenter.py:13-27 on ops.mimo_merge: no dense [M, f, X, Y, Z] volume and no host synchronisation for the
    minimum coordinate; the same features, coordinates and input gradient bit for bit.  One host synchronisation
    (the merged row count)."""
    F_ = in_feat.F
    if not F_.is_cuda:
        return self._pasco_b200_orig_merge(in_feat)
    merged = ops.mimo_merge(F_, in_feat.C)
    if merged is None:                                 # more than 8 subnets, or coordinates the keys cannot hold
        return self._pasco_b200_orig_merge(in_feat)
    feats, coords = merged
    cm = ME.CoordinateManager()                        # unique rows: register the map without the dedup pass
    return ME.SparseTensor(feats, coordinate_map_key=cm._register(coords, 1), coordinate_manager=cm)


def _dense_bottleneck(self, deepest_features, bs, global_min_coords, global_max_coords):
    """unet3d_sparse_v2.py:182-214 on net3d's grid bottleneck: the stride-8 rows densified by rows, the reference's
    SPCDense3Dv2 (dense3d[0]) as box-kernel sparse convolutions on the split-K path, the all-zero rows dropped as
    ME.to_sparse drops them; a SparseTensor on deepest_features' coordinate manager in to_sparse's order.  Four host
    synchronisations, whatever the row count: the grid origin and size, the grid offset's copy from pageable memory,
    and the compaction's row count and error check (plus the kernel maps' construction on the first call at a grid
    size, which net3d.bottleneck_grid caches)."""
    from pasco.models.layers import SPCDense3Dv2
    from pasco.models.unet3d_sparse_v2 import compute_scene_size
    from .net3d import bottleneck_on_grid
    d = self.dense3d
    F_ = deepest_features.F
    if (bs != 1 or not F_.is_cuda or len(d) != 2 or type(d[0]) is not SPCDense3Dv2
            or type(d[1]) is not torch.nn.Dropout3d or (d[1].training and d[1].p > 0)):
        return self._pasco_b200_orig_dense_bottleneck(deepest_features, bs, global_min_coords, global_max_coords)
    scale = deepest_features.tensor_stride[0]
    C_ = deepest_features.C
    gmin = torch.as_tensor(global_min_coords).to(C_.device)
    gmax = torch.max(torch.as_tensor(global_max_coords).to(C_.device), C_[:, 1:].max(dim=0)[0].int())
    scene_size = compute_scene_size(gmin, gmax, scale) // scale
    host = torch.cat([gmin.reshape(3).long(), scene_size.reshape(3).long()]).tolist()       # sync 1
    y, coords = bottleneck_on_grid(d[0], self, F_, C_, scale, host[:3], host[3:])          # syncs 2, 3
    return ME.SparseTensor(y, coords, tensor_stride=scale, coordinate_manager=deepest_features.coordinate_manager)


# ------------------------------------------------------------------------------------------------
# decoder: DecoderBlock.forward (decoder_v3.py:148-172) and DecoderGenerativeSepConvV2's predict_completion_sem_logit
# (:319-394), predict_panop (:396-451) and forward (:453-511) on csrc/decoder.cu and net3d.resize_rows
# ------------------------------------------------------------------------------------------------
DECODER_SYNCS = 3   # host synchronisations of the hooks' own code in one hooked call, at most (see each function); the
                    # reference submodules a hook runs (upsample, process, completion heads, voxel_feats, the
                    # transformer) make their own


def _as_printed(v: int, dev) -> str:
    """How print() shows the reference's 0-dim int64 count on `dev`: its log lines keep their text."""
    return f"tensor({int(v)}, device='{dev}')"


def _resize_channels(resize):
    """C when resize == (MinkowskiBatchNorm(C+3), MinkowskiConvolution(C+3, C, kernel_size=1)), the pair resize_rows
    takes; else None."""
    if not (isinstance(resize, torch.nn.Sequential) and len(resize) == 2):
        return None
    bn, conv = resize[0], resize[1]
    if not (type(conv) is ME.MinkowskiConvolution and conv.use_mm and isinstance(bn, ME.MinkowskiBatchNorm)):
        return None
    C = conv.out_channels
    ok = (bn.bn.num_features == C + 3 and bn.bn.affine and bn.bn.running_mean is not None and conv.in_channels == C + 3)
    return C if ok else None


def _dropout_active(module) -> bool:
    return any(isinstance(m, torch.nn.modules.dropout._DropoutNd) and m.training and m.p > 0
               for m in module.modules())


def _decoder_block_forward(self, x, shortcut, global_min_coords, global_max_coords):
    """decoder_v3.py:148-172 with `resize` as net3d.resize_rows, the function PascoNet's decoder stages call: the split
    BatchNorm, the C feature channels on ops.linear's tensor-core GEMM and the 3 coordinate channels as a rank-3
    update, without concat_coords' (C+3)-channel copy and its new coordinate map.  Host synchronisations of its own:
    the box prune's row count and the shortcut union's."""
    from .net3d import resize_rows
    C = _resize_channels(self.resize)
    if (not x.F.is_cuda or C is None or _dropout_active(self.process)
            or (self.resize[0].bn.training and C % 64 != 0)):
        return self._pasco_b200_orig_forward(x, shortcut, global_min_coords, global_max_coords)
    dec = self.upsample(x)
    c = dec.C
    keep = ((c[:, 1] >= global_min_coords[0]) & (c[:, 1] <= global_max_coords[0])
            & (c[:, 2] >= global_min_coords[1]) & (c[:, 2] <= global_max_coords[1])
            & (c[:, 3] >= global_min_coords[2]) & (c[:, 3] <= global_max_coords[2]))
    dec = self.pruning(dec, keep)
    coords = dec.C[:, 1:].float() / dec.tensor_stride[0]
    y = resize_rows(self.resize[0], self.resize[1], dec.F, coords)
    dec = ME.SparseTensor(y, coordinate_map_key=dec.coordinate_map_key, coordinate_manager=dec.coordinate_manager)
    x = self.process(dec + shortcut)
    return x, [self.completion_heads[str(i)](x) for i in range(self.n_heads)]


def _label_weights(class_frequencies, scale, dev) -> torch.Tensor:
    """decoder_v3.py:353-362: the cap's class weights, float64 on the host, rounded to fp32 as type_as does, moved
    through pinned memory."""
    fr = class_frequencies["1_{}".format(scale)]
    w = fr / np.sum(fr)
    w = np.power(np.amax(w) / w, 1 / 3.0)
    return _on(torch.from_numpy(np.asarray(w)).float(), dev)


_LABEL_DTYPES = (torch.bool, torch.uint8, torch.int16, torch.int32, torch.int64)


def _completion_keep(self, scale, sem_logits, class_frequencies, sem_labels, test):
    """predict_completion_sem_logit on pasco_completion_rows and pasco_topk_mask → the keep mask, or None where the saved
    original decides.  One host synchronisation (every subnet's kept and labelled counts and the rows with a vote),
    and a second one only when a subnet was capped and M >= 3 (the kept union's size)."""
    M = self.n_infers
    if sem_labels is None or not 1 <= M <= 8 or len(sem_logits) < M:
        return None
    Fs = [sem_logits[m].F for m in range(M)]
    n, K = Fs[0].shape
    dev = Fs[0].device
    if not (all(f.is_cuda and f.dtype == torch.float32 and f.shape == Fs[0].shape for f in Fs) and 1 <= K <= 64):
        return None
    try:
        labels = [sem_labels["1_{}".format(scale)][m] for m in range(M)]
        w = None if test else _label_weights(class_frequencies, scale, dev)
    except Exception:
        return None                                   # the original raises where it reads them
    if not all(torch.is_tensor(t) and t.device == dev and t.dtype == labels[0].dtype and t.numel() == labels[0].numel()
               for t in labels) or labels[0].dtype not in _LABEL_DTYPES:
        return None
    probs = [F.softmax(f, dim=-1) for f in Fs]
    _, keep, weight, votes, counts = ops.completion_rows(probs, w, [t.view(torch.uint8) if t.dtype == torch.bool
                                                                   else t for t in labels])
    h = counts.tolist()                                                                      # sync 1
    kept, labelled, bad, n_voted = h[:M], h[M:2 * M], h[2 * M:3 * M], h[3 * M]
    capped = False
    for m in range(M):
        n_m = kept[m]
        if not test and n_m > self.occ_thres[scale] and ((self.training and M <= 2) or M > 3 or n_m > 500000):
            k = int(self.occ_thres[scale])
            if bad[m]:                                # a NaN, inf or negative weight: torch.multinomial's own error
                torch.multinomial(weight[m], k, replacement=False)
            q = torch.empty_like(weight[m]).exponential_(1)       # the draw torch.multinomial makes, same generator
            ops.topk_mask(weight[m], q, k, out=keep[m])
            print("Scale {}, infer {}: ".format(scale, m), _as_printed(n_m, dev), _as_printed(k, dev),
                  _as_printed(labelled[m], dev))
            capped = True
    if capped:
        votes = keep.sum(0)
    out = votes > 0
    thres = self.agg_occ_thres[scale]
    if M >= 3 and not test:
        n_keep = int(out.sum()) if capped else n_voted                                       # sync 2 when capped
        if n_keep <= 2 or n_keep > thres:
            top = torch.topk(votes.long(), k=thres, dim=0)[1]      # massive ties: torch's own tie order, as the original
            out = torch.zeros_like(out).index_fill_(0, top, True)     # `keep[top] = True` without its host copy
            print("Overall keep", _as_printed(n_keep, dev), "after", _as_printed(top.numel(), dev))
    return out


def _predict_completion_sem_logit(self, x, scale, sem_logits, scene_size, min_Cs, max_Cs, class_frequencies,
                                  sem_labels=None, test=False):
    """decoder_v3.py:319-394 without its host reads per subnet, its sorted top-k of the cap and its log lines' device
    tensors: the same keep mask and the same printed lines."""
    keep = _completion_keep(self, scale, sem_logits, class_frequencies, sem_labels, test)
    if keep is None:
        return self._pasco_b200_orig_predict_completion_sem_logit(x, scale, sem_logits, scene_size, min_Cs, max_Cs,
                                                                  class_frequencies, sem_labels=sem_labels, test=test)
    return keep


def _box_on(lo, hi, dev) -> torch.Tensor:
    """int32 [6] = (min_C, max_C) on `dev` without a blocking copy, or None for bounds that are not 3 integers."""
    lo, hi = torch.as_tensor(lo), torch.as_tensor(hi)
    if lo.numel() != 3 or hi.numel() != 3 or lo.dtype.is_floating_point or hi.dtype.is_floating_point:
        return None
    return torch.cat([_on(lo, dev).reshape(3), _on(hi, dev).reshape(3)]).to(torch.int32)


def _predict_panop(self, xs, sem_logits_at_scales, Ts, min_Cs, max_Cs, sem_labels):
    """decoder_v3.py:396-451: every (subnet, scale) crop as one pasco_panop_crop mask and one compaction that serves the
    features and the scale-1 logits, the reference's voxel_feats, pasco_mimo_batch for the padded batches and keep_pad,
    then the reference's transformer_predictor with the original's inputs.  One host synchronisation of its own: all
    crops' counts at once."""
    M = self.n_infers
    args = (xs, sem_logits_at_scales, Ts, min_Cs, max_Cs, sem_labels)
    if sem_labels is None or not 1 <= M <= 8 or 1 not in xs:
        return self._pasco_b200_orig_predict_panop(*args)
    try:
        for m in range(M):
            for s in xs:
                sem_labels["1_{}".format(s)][m]
    except Exception:
        return self._pasco_b200_orig_predict_panop(*args)
    dev = xs[1].F.device
    boxes = [_box_on(min_Cs[m], max_Cs[m], dev) for m in range(M)] if dev.type == "cuda" else [None]
    ok = all(b is not None for b in boxes)
    for s, x in xs.items():
        for m in range(M):
            lg = sem_logits_at_scales[s][m]
            ok = ok and (x.F.is_cuda and x.F.device == dev and lg.F.dtype == torch.float32 and lg.F.device == dev
                         and 1 <= lg.F.shape[1] <= 64 and lg.F.shape[0] == x.F.shape[0]
                         and lg.coordinate_map_key == x.coordinate_map_key)
    if not ok:
        return self._pasco_b200_orig_predict_panop(*args)
    scales = list(xs)
    counts = torch.zeros(M, len(scales), 2, dtype=torch.int32, device=dev)
    masks = {(m, s): ops.panop_crop(sem_logits_at_scales[s][m].F, xs[s].C, boxes[m], counts[m, j])
             for m in range(M) for j, s in enumerate(scales)}
    h = counts.tolist()                                                                      # the one sync
    xs_infers = collections.defaultdict(list)
    sem_logits_pruneds = []
    for m in range(M):
        for j, s in enumerate(scales):
            n_cls, n_keep = h[m][j]
            if n_cls == 0:
                print("line 367: keep.sum() == 0")
            x = xs[s]
            cm = x.coordinate_manager
            kept, _, _ = ops.compact(masks[m, s], n_keep)
            key = cm._register(ops.gather_coords(x.C, kept), x.coordinate_map_key.tensor_stride)
            if s == 1:
                sem_logits_pruneds.append(ME.SparseTensor(ops.GatherRows.apply(sem_logits_at_scales[s][m].F.float(), kept),
                                                          coordinate_map_key=key, coordinate_manager=cm))
            pruned = ME.SparseTensor(ops.GatherRows.apply(x.F.float(), kept), coordinate_map_key=key,
                                     coordinate_manager=cm)
            xs_infers[s].append(self.voxel_feats["scale{}_infer{}".format(s, m)](pruned))
    for s in xs_infers:
        xs_infers[s] = ops.mimo_batch([t.F for t in xs_infers[s]], [t.C for t in xs_infers[s]])[:2]
    batch_F, batch_C, keep_pad = ops.mimo_batch([t.F for t in sem_logits_pruneds], [t.C for t in sem_logits_pruneds],
                                                keep_pad=True)
    panop_predictions = self.transformer_predictor(xs_infers, (batch_F, batch_C), min_Cs, max_Cs, keep_pad)
    return panop_predictions, sem_logits_pruneds


def _decoder_forward(self, x, features, global_min_coords, global_max_coords, min_Cs, max_Cs, class_frequencies, Ts,
                     is_predict_panop=True, sem_labels=None, test=False):
    """decoder_v3.py:453-511 with lines 496-497 as one prune of x and the M logits (net3d.prune_many: one compaction,
    one host synchronisation and one coordinate map per scale where the original makes M + 1).  The pruned tensors
    share that map; their coordinates are identical anyway."""
    from pasco.models import decoder_v3
    from .net3d import prune_many
    if not x.F.is_cuda:
        return self._pasco_b200_orig_forward(x, features, global_min_coords, global_max_coords, min_Cs, max_Cs,
                                             class_frequencies, Ts, is_predict_panop=is_predict_panop,
                                             sem_labels=sem_labels, test=test)
    features = features[::-1]
    sem_logits_at_scales, xs = {}, {}
    for i in range(len(self.dec_blocks)):
        scale = 2 ** (len(self.dec_blocks) - 1 - i)
        x, sem_logits = self.dec_blocks[i](x, features[i], global_min_coords, global_max_coords)
        if scale in [4, 2, 1]:
            scene_size = decoder_v3.compute_scene_size(global_min_coords, global_max_coords)
            keep = self.predict_completion_sem_logit(x, scale, sem_logits, scene_size, min_Cs, max_Cs,
                                                     class_frequencies=class_frequencies, sem_labels=sem_labels,
                                                     test=test)
            if all(c.coordinate_map_key == x.coordinate_map_key and c.F.shape[0] == x.F.shape[0] for c in sem_logits):
                x, sem_logits = prune_many([x] + list(sem_logits), keep)                     # one sync
            else:
                x = self.pruning(x, keep)
                sem_logits = [self.pruning(c, keep) for c in sem_logits]
            xs[scale] = x
            sem_logits_at_scales[scale] = sem_logits
    ret = {"sem_logits_at_scales": sem_logits_at_scales}
    if is_predict_panop:
        panop_predictions, sem_logits_pruneds = self.predict_panop(xs, sem_logits_at_scales, Ts, min_Cs, max_Cs,
                                                                   sem_labels)
        ret["panop_predictions"] = panop_predictions
        ret["sem_logits_pruneds"] = sem_logits_pruneds
    return ret


# ------------------------------------------------------------------------------------------------
# install / uninstall
# ------------------------------------------------------------------------------------------------
_TP = "pasco.models.transformer.transformer_predictor_v2"
_DEC = "pasco.models.decoder_v3"
_NET = "pasco.models.net_panoptic_sparse"
_K360 = "pasco.models.net_panoptic_sparse_kitti360"    # imports pasco.data.kitti360.params, which may not import

# Every hook group in install order: (the trigger modules PASCO_B200_HOOKS waits for, its patch sites).  A site is
# (module, class or None for a module-level name, attribute, replacement, whether the site may be missing); install()
# keeps the original as `_pasco_b200_orig_<attribute>` on that class or module.
_GROUPS = {
    "attention": ((_TP,), (
        (_TP, "TransformerPredictorV2", "forward", _transformer_forward, False),
        ("pasco.models.transformer.blocks", "CrossAttentionLayer", "forward", _cross_attention_forward, False))),
    "postprocess": (("pasco.models.ensembler", "pasco.models.helper"), (      # either Net module imports both
        ("pasco.models.ensembler", "Ensembler", "ensemble_sem_compl", _ensemble_sem_compl, False),
        ("pasco.models.ensembler", "Ensembler", "ensemble_panop", _ensemble_panop, False),
        ("pasco.models.helper", None, "panoptic_inference", _panoptic_inference, False),
        (_NET, None, "panoptic_inference", _panoptic_inference, False),        # the Net modules import it by name
        (_K360, None, "panoptic_inference", _panoptic_inference, True))),
    "evaluate": (("pasco.models.metrics",), (                                   # ... and this one
        (_NET, "Net", "evaluate_all", _evaluate_all, False),
        (_K360, "Net_kitti360", "evaluate_all", _evaluate_all_kitti360, True))),
    "criterion": (("pasco.loss.criterion_sparse", "pasco.loss.losses"), (      # ... and these
        ("pasco.loss.criterion_sparse", "SetCriterion", "compute_losses", _compute_losses, False),
        # the completion losses under the names the Net modules import; pasco.loss.losses keeps its own
        (_NET, None, "compute_sem_compl_loss", _compute_sem_compl_loss, False),
        (_K360, None, "compute_sem_compl_loss_kitti360", _compute_sem_compl_loss_kitti360, True))),
    "trunk": (("pasco.models.augmenter", "pasco.models.unet3d_sparse_v2"), (
        ("pasco.models.unet3d_sparse_v2", "CylinderFeat", "forward", _cylinder_forward, False),
        ("pasco.models.augmenter", "Augmenter", "merge", _augmenter_merge, False),
        ("pasco.models.unet3d_sparse_v2", "UNet3DV2", "dense_bottleneck", _dense_bottleneck, False))),
    "decoder": ((_DEC,), (
        (_DEC, "DecoderBlock", "forward", _decoder_block_forward, False),
        (_DEC, "DecoderGenerativeSepConvV2", "predict_completion_sem_logit", _predict_completion_sem_logit, False),
        (_DEC, "DecoderGenerativeSepConvV2", "predict_panop", _predict_panop, False),
        (_DEC, "DecoderGenerativeSepConvV2", "forward", _decoder_forward, False))),
    "transformer": ((_TP,), (
        ("pasco.models.transformer.position_encoding", "PositionEmbeddingSineSparse", "forward", _pe_forward, False),
        (_TP, "TransformerPredictorV2", "pred_heads", _pred_heads, False))),
}
_installed = set()     # the names of the installed groups


def _owners(sites) -> list:
    """The class or module that holds each site's attribute, None for an optional site that is missing.  Raises when
    any other site's module does not import or lacks the class."""
    out = []
    for module, cls, _, _, optional in sites:
        try:
            mod = importlib.import_module(module)
            out.append(mod if cls is None else getattr(mod, cls))
        except Exception:
            if not optional:
                raise
            out.append(None)
    return out


def _users():
    """The modules that hold the name panoptic_inference: helper and the Net modules, which import it by name (the
    KITTI-360 one when importable)."""
    sites = [site for _, sites in _GROUPS.values() for site in sites if site[2] == "panoptic_inference"]
    return [m for m in _owners(sites) if m is not None]


def install(attention: bool = True, postprocess: bool = False, evaluate: bool = False, criterion: bool = False,
            trunk: bool = False, decoder: bool = False, transformer: bool = False) -> bool:
    """Patch the reference (idempotent per group).  attention: TransformerPredictorV2.forward with its masks as
    bit rows, and the cross-attention layer that takes them; postprocess: the
    Ensembler and panoptic_inference; evaluate: Net.evaluate_all of both Net modules; criterion:
    SetCriterion.compute_losses and the completion losses both Net modules import; trunk: CylinderFeat.forward,
    Augmenter.merge and UNet3DV2.dense_bottleneck; decoder: DecoderBlock.forward and DecoderGenerativeSepConvV2's
    forward, predict_completion_sem_logit and predict_panop; transformer: PositionEmbeddingSineSparse.forward and
    TransformerPredictorV2.pred_heads, and with attention the projections and per-item outputs of the forward.
    Groups install in _GROUPS' order, each only once all its sites have been found.  Returns False at the first
    requested group whose `pasco` modules are not importable; the groups before it stay installed."""
    requested = locals()                               # one keyword per group of _GROUPS
    for group, (_, sites) in _GROUPS.items():
        if not requested[group] or group in _installed:
            continue
        try:
            owners = _owners(sites)
        except Exception:
            return False
        for owner, (_, _, attr, fn, _) in zip(owners, sites):
            if owner is not None:
                setattr(owner, "_pasco_b200_orig_" + attr, getattr(owner, attr))
                setattr(owner, attr, fn)
        _installed.add(group)
    return True


def uninstall() -> None:
    """Restore every attribute install() patched."""
    for group, (_, sites) in _GROUPS.items():
        if group in _installed:
            for owner, (_, _, attr, _, _) in zip(_owners(sites), sites):
                if owner is not None:
                    setattr(owner, attr, getattr(owner, "_pasco_b200_orig_" + attr))
    _installed.clear()


def _parse_groups(value: str) -> frozenset:
    """PASCO_B200_HOOKS: "" / "0" = no group, "1" = the attention group, else a comma list of _GROUPS' names."""
    if value in ("", "0"):
        return frozenset()
    if value == "1":
        return frozenset(list(_GROUPS)[:1])          # the first group: attention
    groups = frozenset(v.strip() for v in value.split(",") if v.strip())
    if not groups <= set(_GROUPS):
        raise ValueError(f"PASCO_B200_HOOKS={value!r}: expected 0, 1 or a comma list of {', '.join(_GROUPS)}")
    return groups


_REQUESTED = _parse_groups(os.environ.get("PASCO_B200_HOOKS", "0"))     # an unknown group raises on import


def _install_requested() -> bool:
    """PASCO_B200_HOOKS: install the requested groups once all their trigger modules have been imported; whether they
    had been.  pasco_b200.me asks on every SparseTensor construction until then."""
    if not all(m in sys.modules for g in _REQUESTED for m in _GROUPS[g][0]):
        return False
    install(**{g: g in _REQUESTED for g in _GROUPS})
    return True
