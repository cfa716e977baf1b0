"""Opt-in hooks that route the UNMODIFIED reference's mask-transformer hot spots onto the sm_90a attention kernels.

The MinkowskiEngine surface (`pasco_b200.me`) already carries every sparse-tensor op of the reference.  Two pieces of
PaSCo's transformer are plain torch in the reference and therefore outside that surface:

  * `CrossAttentionLayer.forward`  (pasco/models/transformer/blocks.py:73-92): `nn.MultiheadAttention` of 100 queries over
    all P voxels — cuBLAS batched GEMMs + a [8, 100, P] softmax volume;
  * `TransformerPredictorV2.compute_attn_mask` (transformer/transformer_predictor_v2.py:220-289): a dense
    [1, 100, X/s, Y/s, Z/s] volume (839 MB at scale 1) built only to be sampled at the key voxels.

`install()` replaces those two methods — at run time, on the imported classes, without touching the reference's files —
with calls into the engine: the attention through ops.cross_attention, which net3d's own decoder uses too (K/V
projections on the wgmma GEMM, the masked softmax·V as `pasco_xattn_forward/backward`: streaming two-pass softmax,
bit-packed mask rows, no [Q, P] score volume in HBM) and the mask as a sparse max-pool + hash look-up.  Same
parameters, same state_dict, same results within the fp32 tolerance (tests/test_dropin_reference.py runs the reference
with and without the hooks).

    import pasco_b200.hooks; pasco_b200.hooks.install()        # after `pasco` is importable, before building Net
    PASCO_B200_HOOKS=1 python scripts/train.py ...              # compat/MinkowskiEngine calls install() lazily
"""
from __future__ import annotations

import torch

from . import me as ME
from . import ops

_installed = False


def _cross_attention_forward(self, q_embed, bb_feat, attn_mask=None, padding_mask=None, pos=None, query_pos=None):
    """blocks.py:73-92 with the attention itself on xattn.cu.  q_embed [B, Q, d]; bb_feat / pos [B, P, d]; attn_mask
    bool [B*heads, Q, P] (True = masked; the reference repeats one [Q, P] mask over the heads)."""
    if padding_mask is not None or not bb_feat.is_cuda:
        return self._pasco_b200_orig_forward(q_embed, bb_feat, attn_mask, padding_mask, pos, query_pos)
    h = self.multihead_attn.num_heads
    q_embed = self.norm(q_embed)
    outs = []
    for b in range(q_embed.shape[0]):
        qb = q_embed[b] if query_pos is None else q_embed[b] + query_pos[b]
        kv = bb_feat[b] if pos is None else bb_feat[b] + pos[b]
        m = attn_mask[b * h] if attn_mask is not None else None    # all heads of an item share one mask
        outs.append(ops.cross_attention(self.multihead_attn, qb, kv, m))
    return q_embed + self.dropout(torch.stack(outs, 0))


def _compute_attn_mask(self, outputs_mask, voxel_coord, src, src_C, src_scale, min_Cs, max_Cs):
    """transformer_predictor_v2.py:220-289 without the dense volume: mask[q, v] = not OR_{u in block_s(v)} (logit[u, q] > 0).
    outputs_mask [B, P1, Q]; voxel_coord [B, P1, 4]; src_C [B, Ps, 4] → bool [B*heads, Q, Ps]."""
    masks = []
    for b in range(outputs_mask.shape[0]):
        keep = (outputs_mask[b].detach() > 0).float().contiguous()               # sigmoid(x) > 0.5
        C1 = voxel_coord[b].to(torch.int32).clone()
        C1[:, 0] = 0
        mgr = ME.CoordinateManager()
        key1, uidx = mgr.insert_and_map(C1.contiguous())                          # padded rows share voxel (0,0,0)
        if uidx is not None:
            keep = ops._gather_rows(keep, uidx)
        if src_scale == 1:
            pooled, pooled_key = keep, key1
        else:
            pooled_key = mgr.stride(key1, src_scale)
            pooled = ops.MaxPoolRows.apply(keep, mgr.pool_map(key1, pooled_key, src_scale), mgr.size(pooled_key))
        Cs = src_C[b].to(torch.int32).clone()
        Cs[:, 0] = 0
        rows = ops.hash_lookup(mgr._table(pooled_key), Cs.contiguous())
        at_keys = ops._gather_rows(pooled.contiguous(), rows)                     # [Ps, Q], zero where no child
        masks.append((at_keys == 0).t())
    m = torch.stack(masks, 0)                                                     # [B, Q, Ps]
    return m.unsqueeze(1).repeat(1, self.nheads, 1, 1).flatten(0, 1)


def install() -> bool:
    """Patch the reference classes (idempotent).  Returns False when `pasco` is not importable."""
    global _installed
    if _installed:
        return True
    try:
        from pasco.models.transformer import blocks
        from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    except Exception:
        return False
    blocks.CrossAttentionLayer._pasco_b200_orig_forward = blocks.CrossAttentionLayer.forward
    blocks.CrossAttentionLayer.forward = _cross_attention_forward
    TransformerPredictorV2._pasco_b200_orig_compute_attn_mask = TransformerPredictorV2.compute_attn_mask
    TransformerPredictorV2.compute_attn_mask = _compute_attn_mask
    _installed = True
    return True


def uninstall() -> None:
    global _installed
    if not _installed:
        return
    from pasco.models.transformer import blocks
    from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    blocks.CrossAttentionLayer.forward = blocks.CrossAttentionLayer._pasco_b200_orig_forward
    TransformerPredictorV2.compute_attn_mask = TransformerPredictorV2._pasco_b200_orig_compute_attn_mask
    _installed = False
