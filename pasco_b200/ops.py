"""Tensor-level wrappers and autograd Functions over the C-ABI (include/pasco_sm100.h).

Everything here runs on CUDA through libpasco_sm100.so; torch supplies device memory, the
current stream and the autograd graph.  Row indices are int32, −1 = no row.
"""
from __future__ import annotations

import ctypes as C
import itertools
import math
import weakref
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import call as _raw_call, ptr, int_array, load


def call(name, *args):
    global CALLS
    CALLS += 1
    _raw_call(name, *args)

_PRECISION = 3          # 3 = bf16x3 split ("fp32" parity mode), 1 = plain bf16 operands
_FORCE_SIMT = False     # validation switch: run every conv on the CUDA-core path
_SIMT_KINDS = None      # validation switch: subset of {'fwd','dgrad','wgrad'} forced onto the CUDA-core path
_SPLIT_K = True          # few-tile / many-offset convs (dense bottleneck) are split over the offsets
_PENDING_STATS = None
_USE_PLANES = True      # gathered convs (K > 1) read pre-split bf16 planes with zero-fill cp.async copies (k_conv_pl /
                        # k_wgrad_pl); False = the round-1 register-gather kernels (kept for cross-checks)
_INFER_FUSION = True    # eval mode without gradients: BatchNorm + activation fused into the planes / the convolution's
                        # inference epilogue (inference_fusion_active); False = the row passes (bit-identical cross-check)
PROFILE = None          # bench.py sets this to a list: (kind, start_event, end_event, meta) per conv launch
PAIR_COUNTS = {}        # nbr.data_ptr() → 0-dim device tensor with the number of valid pairs (profiling only)
CALLS = 0               # number of C-ABI compute calls (each launches >= 1 kernel of ours)


def set_precision(mode) -> None:
    """'fp32' (bf16x3 split operands, ~2^-16 relative) or 'bf16' (single bf16 MMA)."""
    global _PRECISION
    _PRECISION = {"fp32": 3, "bf16": 1, 3: 3, 1: 1}[mode]
    # library ops on the path (cuDNN dense bottleneck, cuBLAS 1x1 convs / projections) follow the same contract:
    # fp32 mode = no TF32 anywhere, bf16 mode = TF32 allowed for the library GEMMs/convs
    torch.backends.cudnn.allow_tf32 = _PRECISION == 1
    torch.backends.cuda.matmul.allow_tf32 = _PRECISION == 1


def get_precision() -> int:
    return _PRECISION


def force_simt(flag: bool, kinds=None) -> None:
    global _FORCE_SIMT, _SIMT_KINDS
    _FORCE_SIMT = bool(flag) and kinds is None
    _SIMT_KINDS = set(kinds) if (flag and kinds is not None) else None


_ERR = {}               # device → int32[1] error flag set by kernels (rows outside a dense volume); read at sync points


def _err_flag(dev) -> torch.Tensor:
    f = _ERR.get(dev)
    if f is None:
        f = _ERR[dev] = torch.zeros(1, dtype=torch.int32, device=dev)
    return f


def raise_pending_errors(dev=None) -> None:
    """Raise what MinkowskiEngine raises immediately (a coordinate outside the dense volume) — called where the host
    already synchronises (compact), and by tests."""
    for d, f in list(_ERR.items()):
        if dev is not None and d != dev:
            continue
        code = int(f.item())
        if code != 0:
            f.zero_()
            if code == 2:
                raise RuntimeError("pasco_b200: a coordinate or batch index lies outside [-32768, 32767] "
                                   "(coordinate keys pack 16 bits per component)")
            raise RuntimeError("pasco_b200: a coordinate lies outside the requested dense volume "
                               "(SparseTensor.dense / to_sparse: check min_coordinate and shape)")


def _i32(t: torch.Tensor) -> torch.Tensor:
    return t if t.dtype == torch.int32 else t.to(torch.int32)


# ----------------------------------------------------------------------------------------------
# hash tables / coordinate maps
# ----------------------------------------------------------------------------------------------
class HashTable:
    """Open-addressing table key(b,x,y,z) → row, resident in HBM."""

    def __init__(self, keys: torch.Tensor, vals: torch.Tensor):
        self.keys, self.vals = keys, vals
        self.capacity = keys.numel()


def _capacity(n: int) -> int:
    cap = 64
    while cap < 2 * n:
        cap <<= 1
    return cap


def hash_insert(coords: torch.Tensor) -> Tuple[HashTable, torch.Tensor]:
    """Insert int32 [N,4] rows.  Returns (table, first_row[N]) — first_row[i] == i iff row i wins."""
    n = coords.shape[0]
    cap = _capacity(n)
    dev = coords.device
    keys = torch.full((cap,), -1, dtype=torch.int64, device=dev)                 # 0xFF… = empty
    vals = torch.full((cap,), 0x7F7F7F7F, dtype=torch.int32, device=dev)
    first = torch.empty(n, dtype=torch.int32, device=dev)
    call("pasco_hash_insert", ptr(coords), n, ptr(keys), ptr(vals), cap, ptr(first), ptr(_err_flag(dev)))
    return HashTable(keys, vals), first


def hash_lookup(table: HashTable, query: torch.Tensor) -> torch.Tensor:
    out = torch.empty(query.shape[0], dtype=torch.int32, device=query.device)
    call("pasco_hash_lookup", ptr(query), query.shape[0], ptr(table.keys), ptr(table.vals), table.capacity, ptr(out))
    return out


def hash_remap(table: HashTable, new_row: torch.Tensor) -> None:
    call("pasco_hash_remap", ptr(table.vals), table.capacity, ptr(new_row))


def coords_floor(coords: torch.Tensor, stride: Sequence[int]) -> torch.Tensor:
    out = torch.empty_like(coords)
    call("pasco_coords_floor", ptr(coords), coords.shape[0], int(stride[0]), int(stride[1]), int(stride[2]), ptr(out))
    return out


def coords_generate_k2(coords: torch.Tensor, out_stride: Sequence[int]) -> torch.Tensor:
    out = torch.empty(coords.shape[0] * 8, 4, dtype=torch.int32, device=coords.device)
    call("pasco_coords_generate_k2", ptr(coords), coords.shape[0], int(out_stride[0]), int(out_stride[1]),
         int(out_stride[2]), ptr(out))
    return out


def kernel_map_probe(out_coords: torch.Tensor, table: HashTable, kernel_size: int, step: Sequence[int]) -> torch.Tensor:
    """nbr[K, N_out] for an odd kernel; step = tensor_stride·dilation per axis."""
    n = out_coords.shape[0]
    nbr = torch.empty(kernel_size ** 3, n, dtype=torch.int32, device=out_coords.device)
    call("pasco_kernel_map_probe", ptr(out_coords), n, ptr(table.keys), ptr(table.vals), table.capacity,
         kernel_size, int(step[0]), int(step[1]), int(step[2]), ptr(nbr))
    return nbr


def kernel_map_box(out_coords: torch.Tensor, table: HashTable, ksize: Sequence[int], step: Sequence[int]) -> torch.Tensor:
    """nbr[kx*ky*kz, N_out] for an anisotropic odd box kernel (offsets x fastest)."""
    n = out_coords.shape[0]
    K = int(ksize[0]) * int(ksize[1]) * int(ksize[2])
    nbr = torch.empty(K, n, dtype=torch.int32, device=out_coords.device)
    call("pasco_kernel_map_box", ptr(out_coords), n, ptr(table.keys), ptr(table.vals), table.capacity,
         int(ksize[0]), int(ksize[1]), int(ksize[2]), int(step[0]), int(step[1]), int(step[2]), ptr(nbr))
    return nbr


def kernel_map_down(child_coords: torch.Tensor, parent_table: HashTable, n_parent: int, ks: int,
                    child_stride: Sequence[int], want_nbr: bool = True):
    n = child_coords.shape[0]
    dev = child_coords.device
    parent_of = torch.empty(n, dtype=torch.int32, device=dev)
    slot_of = torch.empty(n, dtype=torch.int32, device=dev)
    nbr = torch.full((ks ** 3, n_parent), -1, dtype=torch.int32, device=dev) if want_nbr else None
    call("pasco_kernel_map_down", ptr(child_coords), n, ptr(parent_table.keys), ptr(parent_table.vals),
         parent_table.capacity, ks, int(child_stride[0]), int(child_stride[1]), int(child_stride[2]),
         ptr(parent_of), ptr(slot_of), ptr(nbr), n_parent)
    return parent_of, slot_of, nbr


# ----------------------------------------------------------------------------------------------
# order-preserving compaction
# ----------------------------------------------------------------------------------------------
def compact(mask: torch.Tensor, total: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """mask bool/uint8 [N] → (kept_rows[int32 N'], new_row[int32 N], N').  One host sync (N'), none when the caller
    already knows N' and passes it as `total`."""
    n = mask.shape[0]
    dev = mask.device
    m8 = mask.to(torch.uint8) if mask.dtype != torch.uint8 else mask
    m8 = m8.contiguous()
    if n == 0:
        z = torch.zeros(0, dtype=torch.int32, device=dev)
        return z, z, 0
    nb = (n + 1023) // 1024
    counts = torch.empty(nb, dtype=torch.int32, device=dev)
    call("pasco_mask_block_counts", ptr(m8), n, ptr(counts))
    incl = torch.cumsum(counts, 0, dtype=torch.int32)       # ≤ ~1k elements: plumbing
    offsets = (incl - counts).contiguous()
    if total is None:
        total = int(incl[-1].item())
        if _ERR:
            raise_pending_errors(dev)
    new_row = torch.empty(n, dtype=torch.int32, device=dev)
    kept = torch.empty(total, dtype=torch.int32, device=dev)
    call("pasco_mask_compact", ptr(m8), n, ptr(offsets), ptr(new_row), ptr(kept))
    return kept, new_row, total


def gather_coords(coords: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    out = torch.empty(rows.shape[0], 4, dtype=torch.int32, device=coords.device)
    call("pasco_gather_coords", ptr(coords), ptr(rows), rows.shape[0], ptr(out))
    return out


def _gather_rows(src: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    out = torch.empty(rows.shape[0], src.shape[1], dtype=torch.float32, device=src.device)
    call("pasco_gather_rows", ptr(src), ptr(rows), rows.shape[0], src.shape[1], ptr(out))
    return out


def _scatter_rows(src: torch.Tensor, rows: torch.Tensor, dst: torch.Tensor, accumulate: bool) -> None:
    call("pasco_scatter_rows", ptr(src), ptr(rows), rows.shape[0], src.shape[1], ptr(dst), int(accumulate))


class GatherRows(torch.autograd.Function):
    """out[r] = src[rows[r]] (rows unique or −1).  Backward scatters into a zero tensor."""

    @staticmethod
    def forward(ctx, src, rows):
        ctx.save_for_backward(rows)
        ctx.n_src = src.shape[0]
        return _gather_rows(src.contiguous().float(), rows)

    @staticmethod
    def backward(ctx, g):
        (rows,) = ctx.saved_tensors
        gin = torch.zeros(ctx.n_src, g.shape[1], dtype=torch.float32, device=g.device)
        _scatter_rows(g.contiguous(), rows, gin, False)
        return gin, None


class UnionAdd(torch.autograd.Function):
    """out = zeros[N_out]; out[:N_a] = a; out[rows_b] += b   (coordinate-union add, decoder_v3.py:163)."""

    @staticmethod
    def forward(ctx, a, b, rows_b, n_out):
        ctx.save_for_backward(rows_b)
        ctx.na = a.shape[0]
        out = torch.zeros(n_out, a.shape[1], dtype=torch.float32, device=a.device)
        out[: a.shape[0]].copy_(a)
        _scatter_rows(b.contiguous(), rows_b, out, True)
        return out

    @staticmethod
    def backward(ctx, g):
        (rows_b,) = ctx.saved_tensors
        g = g.contiguous()
        return g[: ctx.na], _gather_rows(g, rows_b), None, None


# ----------------------------------------------------------------------------------------------
# dense <-> sparse
# ----------------------------------------------------------------------------------------------
def _geom(min_c, stride):
    return int_array(min_c), int_array(stride)


class ToDense(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feats, coords, min_c, stride, shape):
        B, Cc, X, Y, Z = shape
        dense = torch.zeros(shape, dtype=torch.float32, device=feats.device)
        mc, st = _geom(min_c, stride)
        call("pasco_to_dense", ptr(feats.contiguous()), ptr(coords), feats.shape[0], Cc, mc, st, ptr(dense), B, X, Y, Z,
             ptr(_err_flag(feats.device)))
        ctx.save_for_backward(coords)
        ctx.meta = (tuple(min_c), tuple(stride), tuple(shape))
        return dense

    @staticmethod
    def backward(ctx, g):
        (coords,) = ctx.saved_tensors
        min_c, stride, shape = ctx.meta
        return from_dense_raw(g.contiguous(), coords, min_c, stride), None, None, None, None


def from_dense_raw(dense: torch.Tensor, coords: torch.Tensor, min_c, stride) -> torch.Tensor:
    B, Cc, X, Y, Z = dense.shape
    feats = torch.empty(coords.shape[0], Cc, dtype=torch.float32, device=dense.device)   # out-of-volume rows read as 0
    mc, st = _geom(min_c, stride)
    call("pasco_from_dense", ptr(dense), ptr(coords), coords.shape[0], Cc, mc, st, ptr(feats), B, X, Y, Z,
         ptr(_err_flag(dense.device)))
    return feats


class FromDense(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dense, coords, min_c, stride):
        ctx.save_for_backward(coords)
        ctx.meta = (tuple(min_c), tuple(stride), tuple(dense.shape))
        return from_dense_raw(dense.contiguous().float(), coords, min_c, stride)

    @staticmethod
    def backward(ctx, g):
        (coords,) = ctx.saved_tensors
        min_c, stride, shape = ctx.meta
        B, Cc, X, Y, Z = shape
        dense = torch.zeros(shape, dtype=torch.float32, device=g.device)
        mc, st = _geom(min_c, stride)
        call("pasco_to_dense", ptr(g.contiguous()), ptr(coords), g.shape[0], Cc, mc, st, ptr(dense), B, X, Y, Z, None)
        return dense, None, None, None


def dense_occupancy(dense: torch.Tensor) -> torch.Tensor:
    B, Cc = dense.shape[:2]
    cells = dense[0, 0].numel()
    mask = torch.empty(B * cells, dtype=torch.uint8, device=dense.device)
    call("pasco_dense_occupancy", ptr(dense), B, Cc, cells, ptr(mask))
    return mask


# ----------------------------------------------------------------------------------------------
# sparse convolution
# ----------------------------------------------------------------------------------------------
class KernelMap:
    """Neighbour tables of one (in_map, out_map, kernel) triple, both directions.

    nbr   int32 [K, N_out]: input row feeding output row o through offset k (forward / wgrad)
    nbr_t int32 [K, N_in] : output row fed by input row i, table row k' using weight slice koff_t[k']
    """

    def __init__(self, nbr, n_in, n_out, nbr_t=None, koff_t=None, build_t=None):
        self.nbr, self.n_in, self.n_out = nbr, n_in, n_out
        if PROFILE is not None:
            PAIR_COUNTS[nbr.data_ptr()] = (nbr >= 0).sum()
        self._nbr_t, self._koff_t, self._build_t = nbr_t, koff_t, build_t
        self.K = nbr.shape[0]

    def transposed(self):
        if self._nbr_t is None:
            self._nbr_t, self._koff_t = self._build_t()
        return self._nbr_t, self._koff_t


class PackedWeights:
    """Tensor-core shared-memory images of one weight tensor (forward and transposed), owned by the module
    that owns the parameter and re-packed whenever the parameter changes (optimizer step, load_state_dict,
    device move).  Keyed by (data_ptr, version, shape) of that one parameter only."""

    def __init__(self):
        self._slots = {}

    def get(self, weight: torch.Tensor, transpose: bool) -> torch.Tensor:
        tag = (weight.data_ptr(), weight._version, tuple(weight.shape))
        hit = self._slots.get(transpose)
        if hit is not None and hit[0] == tag:
            return hit[1]
        K, Cin, Cout = weight.shape
        nbytes = _lib.load().pasco_conv_packed_bytes(K, Cin, Cout)
        buf = torch.empty(nbytes, dtype=torch.uint8, device=weight.device)
        call("pasco_conv_pack_weights", ptr(weight.detach().contiguous()), K, Cin, Cout, int(transpose), ptr(buf))
        self._slots[transpose] = (tag, buf)
        return buf


def use_planes(flag: bool) -> None:
    global _USE_PLANES
    _USE_PLANES = bool(flag)


def split_planes(x: torch.Tensor, scale=None, shift=None, act: int = 0):
    """x fp32 [N,C] → (hi, lo) bf16 planes [N,C] of act(x*scale+shift) with x ≈ hi + lo; lo is None in bf16 mode."""
    n, c = x.shape
    hi = torch.empty(n, c, dtype=torch.bfloat16, device=x.device)
    lo = torch.empty(n, c, dtype=torch.bfloat16, device=x.device) if _PRECISION == 3 else None
    call("pasco_split_planes", ptr(x), n, c, 0, ptr(scale), ptr(shift), act, ptr(hi), ptr(lo))
    return hi, lo


def conv_path(kind: str, c_contract: int, c_out: int, K: int, nbr, n_rows: int) -> str:
    """The kernels one convolution launch runs on: 'planes' (pasco_conv_forward_planes / pasco_conv_wgrad_planes),
    'splitk' (pasco_conv_forward_splitk), 'regs' (pasco_conv_forward_tc / pasco_conv_wgrad_tc) or 'simt' (CUDA cores).
    kind 'fwd' / 'dgrad': c_contract gathered channels → c_out channels of n_rows output rows through K offsets of the
    neighbour table nbr (None: identity rows); 'wgrad': c_contract = Cin, c_out = Cout (never split, n_rows unused).
    The tensor-core kernels take both channel counts as multiples of 16 and c_out <= 512."""
    if _FORCE_SIMT or (_SIMT_KINDS is not None and kind in _SIMT_KINDS):
        return "simt"
    if c_contract % 16 or c_contract < 16 or c_out % 16 or not 16 <= c_out <= 512:
        return "simt"
    if kind != "wgrad":
        if K > 1024:
            return "simt"
        if _SPLIT_K and load().pasco_conv_splitk_workspace_bytes(K, n_rows, c_out) > 0:
            return "splitk"
    return "planes" if _USE_PLANES and nbr is not None and K > 1 else "regs"


def conv_apply(feats: torch.Tensor, weight: torch.Tensor, nbr: Optional[torch.Tensor], n_out: int,
               transpose_w: bool, koff: Optional[Sequence[int]], bias: Optional[torch.Tensor] = None,
               packs: Optional[PackedWeights] = None, want_stats: bool = False, planes=None,
               planes_out: Optional[list] = None) -> torch.Tensor:
    """out[o] = Σ_k feats[nbr[k,o]] @ Wk, Wk = W[koff[k]] (transposed when transpose_w).
    want_stats: the kernel's epilogue also accumulates the column sums / sums of squares of `out` (the training-mode
    BatchNorm statistics of the layer that follows) and leaves them for BatchNormAct (see take_pending_stats).
    planes: (hi, lo) bf16 planes of the gathered rows if the caller already has them (BNActConv passes the planes of
    act(BN(x))); planes_out: a list that receives the planes this call made (the backward pass reuses them for the
    weight gradient)."""
    K, Cin, Cout = weight.shape
    c_contract, c_out = (Cout, Cin) if transpose_w else (Cin, Cout)
    assert feats.shape[1] == c_contract
    feats = feats.contiguous()
    out = torch.empty(n_out, c_out, dtype=torch.float32, device=feats.device)
    kk = nbr.shape[0] if nbr is not None else 1
    koff_arr = int_array(koff) if koff is not None else None
    prof = PROFILE
    if prof is not None:
        ev0 = torch.cuda.Event(enable_timing=True)
        ev0.record()
    global _PENDING_STATS
    _PENDING_STATS = None            # statistics of an earlier launch never survive another convolution
    path = conv_path("dgrad" if transpose_w else "fwd", c_contract, c_out, kk, nbr, n_out)
    stats = None
    if want_stats and path in ("planes", "regs") and n_out >= 4096:
        stats = torch.zeros(2, c_out, dtype=torch.float64, device=feats.device)
    if path == "planes":
        hi, lo = planes if planes is not None else split_planes(feats)
        if planes_out is not None:
            planes_out.append((hi, lo))
        call("pasco_conv_forward_planes", ptr(hi), ptr(lo), feats.shape[0], ptr(nbr), kk, n_out, c_contract, c_out,
             ptr((packs or PackedWeights()).get(weight, transpose_w)), koff_arr, ptr(bias), ptr(stats), ptr(out),
             _PRECISION, 0, 0)
    elif path == "splitk":
        ws_bytes = load().pasco_conv_splitk_workspace_bytes(kk, n_out, c_out)
        ws = torch.empty(ws_bytes // 4, dtype=torch.float32, device=feats.device)
        call("pasco_conv_forward_splitk", ptr(feats), feats.shape[0], ptr(nbr), kk, n_out, c_contract, c_out,
             ptr((packs or PackedWeights()).get(weight, transpose_w)), koff_arr, ptr(bias), ptr(out), _PRECISION, 0, 0,
             ptr(ws), ws_bytes)
    elif path == "regs":
        call("pasco_conv_forward_tc", ptr(feats), feats.shape[0], ptr(nbr), kk, n_out, c_contract, c_out,
             ptr((packs or PackedWeights()).get(weight, transpose_w)), koff_arr, ptr(bias), ptr(stats), ptr(out),
             _PRECISION, 0, 0)
    else:
        if nbr is None:
            nbr = torch.arange(n_out, dtype=torch.int32, device=feats.device).view(1, -1)
        call("pasco_conv_forward_simt", ptr(feats), ptr(nbr), kk, n_out, c_contract, c_out,
             ptr(weight.detach().contiguous()), int(transpose_w), koff_arr, ptr(bias), ptr(out))
    if prof is not None:
        ev1 = torch.cuda.Event(enable_timing=True)
        ev1.record()
        prof.append(("dgrad" if transpose_w else "fwd", ev0, ev1,
                     dict(n_in=feats.shape[0], n_out=n_out, K=kk, Cin=c_contract, Cout=c_out,
                          pairs=PAIR_COUNTS.get(nbr.data_ptr()) if nbr is not None else None,
                          tc=path != "simt", precision=_PRECISION, path=path)))
    if stats is not None:
        _PENDING_STATS = (weakref.ref(out), out.data_ptr(), out._version, tuple(out.shape), stats)
    return out


def conv_infer(planes, weight: torch.Tensor, bias: Optional[torch.Tensor], kmap: KernelMap,
               packs: Optional[PackedWeights] = None, residual: Optional[torch.Tensor] = None, act_out: int = 0,
               want_out: bool = True, next_coefs=None, next_act: int = 0, want_next: bool = False):
    """Grad-free forward of a stride-1 plane-path convolution on the inference epilogue
    (pasco_conv_forward_planes_infer): from the planes (hi, lo) of the gathered input,
        v = conv + bias;  v = act_out(residual + v) when a residual is given
    and returns (out, next_planes): out = v as fp32 [n_out, Cout] when want_out (else None), next_planes = the bf16 planes
    of act_next(v * scale + shift) with (scale, shift) = next_coefs (the next layer's eval BatchNorm, bn_eval_coefs; None =
    no affine) when want_next (else None).  Bit for bit what conv_apply, affine_act and split_planes compute in turn, in
    one launch and without the fp32 intermediates or the statistics."""
    if torch.is_grad_enabled():
        raise RuntimeError("ops.conv_infer records no autograd graph: call it under torch.no_grad()")
    K, Cin, Cout = weight.shape
    if conv_path("fwd", Cin, Cout, kmap.K, kmap.nbr, kmap.n_out) != "planes":
        raise RuntimeError(f"ops.conv_infer: a {Cin}->{Cout} convolution over {kmap.K} offsets is not on the plane-gather path")
    hi, lo = planes
    n, dev = kmap.n_out, hi.device
    out = torch.empty(n, Cout, dtype=torch.float32, device=dev) if want_out else None
    nhi = torch.empty(n, Cout, dtype=torch.bfloat16, device=dev) if want_next else None
    nlo = torch.empty(n, Cout, dtype=torch.bfloat16, device=dev) if want_next and _PRECISION == 3 else None
    scale, shift = (c.contiguous() for c in next_coefs) if next_coefs is not None else (None, None)
    if residual is not None:
        residual = residual.contiguous()
        assert residual.shape == (n, Cout) and residual.dtype == torch.float32
    prof = PROFILE
    if prof is not None:
        ev0 = torch.cuda.Event(enable_timing=True)
        ev0.record()
    global _PENDING_STATS
    _PENDING_STATS = None
    call("pasco_conv_forward_planes_infer", ptr(hi), ptr(lo), hi.shape[0], ptr(kmap.nbr), kmap.K, n, Cin, Cout,
         ptr((packs or PackedWeights()).get(weight, False)), None, ptr(bias.view(-1).contiguous() if bias is not None else None),
         ptr(residual), act_out, ptr(out), ptr(scale), ptr(shift), next_act, ptr(nhi), ptr(nlo), _PRECISION, 0)
    if prof is not None:
        ev1 = torch.cuda.Event(enable_timing=True)
        ev1.record()
        prof.append(("fwd", ev0, ev1, dict(n_in=hi.shape[0], n_out=n, K=kmap.K, Cin=Cin, Cout=Cout,
                                           pairs=PAIR_COUNTS.get(kmap.nbr.data_ptr()), tc=True, precision=_PRECISION,
                                           path="planes_infer")))
    return out, ((nhi, nlo) if want_next else None)


def take_pending_stats(x: torch.Tensor) -> Optional[torch.Tensor]:
    """Column statistics a convolution epilogue produced for exactly this tensor (same storage, shape and version —
    any in-place change since bumps the version), or None.  Consumed once."""
    global _PENDING_STATS
    pend, _PENDING_STATS = _PENDING_STATS, None
    if pend is None:
        return None
    ref, dptr, ver, shape, stats = pend
    # the producing tensor must still be alive (a freed block re-used at the same address is another tensor) and x must
    # be that storage, unmodified
    if ref() is not None and dptr == x.data_ptr() and ver == x._version and shape == tuple(x.shape):
        return stats
    return None


def split_k(flag: bool) -> None:
    global _SPLIT_K
    _SPLIT_K = bool(flag)


def conv_wgrad(feats: torch.Tensor, gout: torch.Tensor, nbr: Optional[torch.Tensor], K: int, Cin: int, Cout: int,
               in_planes=None, g_planes=None) -> torch.Tensor:
    """in_planes / g_planes: (hi, lo) bf16 planes of the gathered rows and of gout when the caller has them (the forward
    pass made the former, the backward pass splits the latter once for the input and the weight gradient)."""
    n_out = gout.shape[0]
    dW = torch.zeros(K, Cin, Cout, dtype=torch.float32, device=feats.device)
    feats, gout = feats.contiguous(), gout.contiguous()
    prof = PROFILE
    if prof is not None:
        ev0 = torch.cuda.Event(enable_timing=True)
        ev0.record()
    path = conv_path("wgrad", Cin, Cout, K, nbr, n_out)
    if path == "planes":
        ih, il = in_planes if in_planes is not None else split_planes(feats)
        gh, gl = g_planes if g_planes is not None else split_planes(gout)
        call("pasco_conv_wgrad_planes", ptr(ih), ptr(il), feats.shape[0], ptr(nbr), K, n_out, Cin, Cout, ptr(gh), ptr(gl),
             ptr(dW), _PRECISION, 0, 0)
    elif path == "regs":
        call("pasco_conv_wgrad_tc", ptr(feats), feats.shape[0], ptr(nbr), K, n_out, Cin, Cout, ptr(gout), ptr(dW),
             _PRECISION, 0, 0)
    else:
        if nbr is None:
            nbr = torch.arange(n_out, dtype=torch.int32, device=feats.device).view(1, -1)
        call("pasco_conv_wgrad_simt", ptr(feats), ptr(nbr), K, n_out, Cin, Cout, ptr(gout), ptr(dW))
    if prof is not None:
        ev1 = torch.cuda.Event(enable_timing=True)
        ev1.record()
        prof.append(("wgrad", ev0, ev1, dict(n_in=feats.shape[0], n_out=n_out, K=K, Cin=Cin, Cout=Cout,
                                             pairs=PAIR_COUNTS.get(nbr.data_ptr()) if nbr is not None else None,
                                             tc=path != "simt", precision=_PRECISION, path=path)))
    return dW


class SparseConv(torch.autograd.Function):
    """ME ConvolutionForward/Backward over a cached KernelMap."""

    @staticmethod
    def forward(ctx, feats, weight, bias, kmap: KernelMap, packs: Optional[PackedWeights] = None):
        ctx.kmap = kmap
        ctx.packs = packs
        ctx.has_bias = bias is not None
        made = []
        out = conv_apply(feats, weight, kmap.nbr, kmap.n_out, False, None,
                         bias.view(-1).contiguous() if bias is not None else None, packs=packs, want_stats=True,
                         planes_out=made)
        # the weight gradient gathers the same rows: keep the planes the forward made instead of splitting again
        ctx.n_planes = 0
        if made and weight.requires_grad:
            hi, lo = made[0]
            ctx.n_planes = 1 if lo is None else 2
            ctx.save_for_backward(feats, weight, *([hi] if lo is None else [hi, lo]))
        else:
            ctx.save_for_backward(feats, weight)
        return out

    @staticmethod
    def backward(ctx, g):
        feats, weight = ctx.saved_tensors[:2]
        in_planes = None
        if ctx.n_planes:
            in_planes = (ctx.saved_tensors[2], ctx.saved_tensors[3] if ctx.n_planes == 2 else None)
        kmap: KernelMap = ctx.kmap
        g = g.contiguous()
        gin = gw = gb = None
        K, Cin, Cout = weight.shape
        g_planes = None
        if ctx.needs_input_grad[0] and ctx.needs_input_grad[1] and "planes" in (
                conv_path("dgrad", Cout, Cin, K, kmap.nbr, kmap.n_in), conv_path("wgrad", Cin, Cout, K, kmap.nbr, kmap.n_out)):
            g_planes = split_planes(g)          # one split of the output gradient serves dgrad (gather) and wgrad (B operand)
        if ctx.needs_input_grad[0]:
            nbr_t, koff_t = kmap.transposed()
            gin = conv_apply(g, weight, nbr_t, kmap.n_in, True, koff_t, packs=ctx.packs, planes=g_planes)
        if ctx.needs_input_grad[1]:
            gw = conv_wgrad(feats, g, kmap.nbr, K, Cin, Cout, in_planes=in_planes, g_planes=g_planes)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = g.sum(0, keepdim=True)
        return gin, gw, gb, None, None


# ----------------------------------------------------------------------------------------------
# pooling / reductions
# ----------------------------------------------------------------------------------------------
class MaxPoolRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feats, parent_of, n_parent):
        feats = feats.contiguous()
        out = torch.full((n_parent, feats.shape[1]), float("-inf"), dtype=torch.float32, device=feats.device)
        call("pasco_maxpool_forward", ptr(feats), ptr(parent_of), feats.shape[0], feats.shape[1], ptr(out))
        ctx.save_for_backward(feats, parent_of, out)
        return out

    @staticmethod
    def backward(ctx, g):
        feats, parent_of, out = ctx.saved_tensors
        p = parent_of.long()
        hit = feats == out[p]
        return torch.where(hit, g[p], torch.zeros_like(feats)), None, None


class ScatterMax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, src, index, n_seg):
        src = src.contiguous().float()
        index = index.contiguous().long()
        out = torch.full((n_seg, src.shape[1]), float("-inf"), dtype=torch.float32, device=src.device)
        arg = torch.full((n_seg, src.shape[1]), src.shape[0], dtype=torch.int64, device=src.device)
        call("pasco_scatter_max", ptr(src), ptr(index), src.shape[0], src.shape[1], ptr(out), n_seg, ptr(arg))
        ctx.save_for_backward(arg)
        ctx.n_src = src.shape[0]
        ctx.mark_non_differentiable(arg)
        return out, arg

    @staticmethod
    def backward(ctx, g, _):
        (arg,) = ctx.saved_tensors
        gsrc = torch.zeros(ctx.n_src + 1, g.shape[1], dtype=g.dtype, device=g.device)
        gsrc.scatter_(0, arg, g)            # arg == n_src for empty segments → dummy row
        return gsrc[: ctx.n_src], None, None


def scatter_max(src: torch.Tensor, index: torch.Tensor, dim: int = 0, out=None, dim_size: Optional[int] = None):
    """torch_scatter.scatter_max(src[P,C], index[P], dim=0) → (values, argmax); empty segments → 0
    (pasco/models/unet3d_sparse_v2.py:79)."""
    if dim != 0 or src.ndim != 2 or out is not None:
        raise NotImplementedError("pasco_b200.scatter_max: only src[P,C], dim=0 is on PaSCo's path")
    n_seg = int(index.max().item()) + 1 if dim_size is None else int(dim_size)
    return ScatterMax.apply(src, index, n_seg)


# ----------------------------------------------------------------------------------------------
# point voxeliser grouping and the MIMO merge (csrc/voxel.cu)
# ----------------------------------------------------------------------------------------------
def voxel_group(rows: torch.Tensor) -> Optional[Tuple[torch.Tensor, torch.Tensor]]:
    """torch.unique(rows, dim=0, return_inverse=True) for int32 / int64 (b, x, y, z) rows [P, 4], bit for bit: (unique
    rows [U, 4] of rows' dtype in ascending lexicographic order, int64 inverse [P]).  None when a component lies
    outside [-32768, 32767] (the packed keys cannot hold it).  One host synchronisation (U and the range flag)."""
    if rows.dtype not in (torch.int32, torch.int64) or rows.ndim != 2 or rows.shape[1] != 4:
        raise ValueError("voxel_group takes int32 or int64 [P, 4] rows")
    rows = rows.contiguous()
    n, dev, is64 = rows.shape[0], rows.device, int(rows.dtype == torch.int64)
    if n == 0:
        return rows.new_zeros(0, 4), torch.zeros(0, dtype=torch.int64, device=dev)
    cap = _capacity(n)
    keys = torch.full((cap,), -1, dtype=torch.int64, device=dev)
    ukeys = torch.empty(n, dtype=torch.int64, device=dev)
    stats = torch.zeros(2, dtype=torch.int32, device=dev)
    call("pasco_voxel_group", ptr(rows), is64, n, ptr(keys), cap, ptr(ukeys), ptr(stats))
    U, bad = stats.tolist()
    if bad:
        return None
    vals = torch.empty(cap, dtype=torch.int32, device=dev)
    unq = torch.empty(U, 4, dtype=rows.dtype, device=dev)
    inv = torch.empty(n, dtype=torch.int64, device=dev)
    call("pasco_voxel_group_order", ptr(rows), is64, n, ptr(keys), ptr(vals), cap, ptr(ukeys), U, ptr(unq), ptr(inv))
    return unq, inv


class MimoMerge(torch.autograd.Function):
    """Augmenter.merge on the cells of pasco_mimo_merge_cells: (features [U, M·f], coordinates [U, 4]); the backward
    gathers the features' gradient back to the input rows."""

    @staticmethod
    def forward(ctx, F, coords, M, cells):
        keys, vals, cap, ukeys, U = cells
        n, f = F.shape
        out_c = torch.empty(U, 4, dtype=torch.int32, device=F.device)
        out = torch.empty(U, M * f, dtype=torch.float32, device=F.device)
        row_of = torch.empty(n, dtype=torch.int32, device=F.device)
        call("pasco_mimo_merge_forward", ptr(coords), ptr(F), n, f, M, ptr(keys), ptr(vals), cap, ptr(ukeys), U,
             ptr(out_c), ptr(out), ptr(row_of))
        ctx.save_for_backward(coords, row_of)
        ctx.M = M
        ctx.mark_non_differentiable(out_c)
        return out, out_c

    @staticmethod
    def backward(ctx, g, _):
        coords, row_of = ctx.saved_tensors
        n = coords.shape[0]
        f = g.shape[1] // ctx.M
        gin = torch.empty(n, f, dtype=torch.float32, device=g.device)
        call("pasco_mimo_merge_backward", ptr(coords), ptr(row_of), n, f, ctx.M, ptr(g.contiguous().float()), ptr(gin))
        return gin, None, None, None


def mimo_merge(F: torch.Tensor, coords: torch.Tensor, max_subnets: int = 8):
    """Augmenter.merge (augmenter.py:13-27) on the rows, without the dense volume: F fp32 [n, f], coords int [n, 4] with
    the subnet index t in the batch column → (features [U, M·f] with subnet t's channels at t·f, int32 coordinates
    [U, 4] = (0, x, y, z)), M = largest t + 1, the cells in ascending (x, y, z) order, cells whose M·f features are all
    ±0 dropped as ME.to_sparse drops them.  Bit-identical to the dense path, forward and backward.  None for more than
    `max_subnets` subnets, a negative t or a coordinate outside [-32768, 32767].  One host synchronisation (U, M and
    the range flag); none for the minimum coordinate."""
    coords = _i32(coords).contiguous()
    n, f, dev = F.shape[0], F.shape[1], F.device
    if n == 0:
        return None
    Fc = F.contiguous().float()
    cap = _capacity(n)
    keys = torch.full((cap,), -1, dtype=torch.int64, device=dev)
    vals = torch.zeros(cap, dtype=torch.int32, device=dev)
    ukeys = torch.empty(n, dtype=torch.int64, device=dev)
    stats = torch.zeros(3, dtype=torch.int32, device=dev)
    call("pasco_mimo_merge_cells", ptr(coords), ptr(Fc.detach()), n, f, ptr(keys), ptr(vals), cap, ptr(ukeys),
         ptr(stats))
    U, top, bad = stats.tolist()
    M = top + 1
    if bad or M > max_subnets:
        return None
    return MimoMerge.apply(Fc, coords, M, (keys, vals, cap, ukeys, U))


# ----------------------------------------------------------------------------------------------
# the reference decoder's glue (csrc/decoder.cu)
# ----------------------------------------------------------------------------------------------
def _ptrs(ts) -> C.Array:
    return (C.c_void_p * len(ts))(*[ptr(t) for t in ts])


def completion_rows(probs: List[torch.Tensor], w: Optional[torch.Tensor] = None,
                    labels: Optional[List[torch.Tensor]] = None):
    """predict_completion_sem_logit's per-row pass (decoder_v3.py:333-345) over the M subnets' softmax rows [N, K]
    (M <= 8, K <= 64): (cls int32 [M, N], keep bool [M, N], weight fp32 [M, N] = p_max · w[cls] or None without w,
    votes int32 [N], counts int32 [3M + 1] = kept rows per subnet, labelled cells per subnet, rows per subnet whose
    weight is not a finite value >= 0, rows with a vote).  labels: M device volumes of one integer dtype."""
    M, (n, K) = len(probs), probs[0].shape
    dev = probs[0].device
    probs = [p.contiguous() for p in probs]
    cls = torch.empty(M, n, dtype=torch.int32, device=dev)
    keep = torch.empty(M, n, dtype=torch.bool, device=dev)
    weight = torch.empty(M, n, dtype=torch.float32, device=dev) if w is not None else None
    votes = torch.empty(n, dtype=torch.int32, device=dev)
    counts = torch.zeros(3 * M + 1, dtype=torch.int32, device=dev)
    labels = None if labels is None else [t.contiguous() for t in labels]
    call("pasco_completion_rows", _ptrs(probs), M, n, K, ptr(w), _ptrs(labels) if labels else None,
         labels[0].numel() if labels else 0, labels[0].element_size() if labels else 1, ptr(cls), ptr(keep),
         ptr(weight), ptr(votes), ptr(counts))
    return cls, keep, weight, votes, counts


def topk_mask(w: torch.Tensor, q: torch.Tensor, k: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """bool [N]: the k largest w / q (fp32, IEEE division), ties at the k-th value taken by lowest row.  With q drawn as
    torch.multinomial draws it (torch.empty_like(w).exponential_(1) on the same generator), the row set of
    torch.multinomial(w, k, replacement=False), without its sort.  w >= 0 and finite; 1 <= k <= N."""
    keep = torch.empty(w.shape[0], dtype=torch.bool, device=w.device) if out is None else out
    call("pasco_topk_mask", ptr(w.contiguous()), ptr(q.contiguous()), w.shape[0], int(k), ptr(keep))
    return keep


def panop_crop(logits: torch.Tensor, coords: torch.Tensor, box: torch.Tensor, counts: torch.Tensor) -> torch.Tensor:
    """predict_panop's prunes of one subnet and scale as one mask (decoder_v3.py:409-434): bool [N] = argmax != 0 and
    box[:3] <= (x, y, z) <= box[3:], or the first 1000 rows inside the box when no argmax is != 0.  counts int32 [2]
    (zeroed): rows with argmax != 0, rows kept.  No host synchronisation."""
    mask = torch.empty(logits.shape[0], dtype=torch.bool, device=logits.device)
    call("pasco_panop_crop", ptr(logits.contiguous()), logits.shape[0], logits.shape[1], ptr(_i32(coords).contiguous()),
         ptr(box), ptr(mask), ptr(counts))
    return mask


class MimoBatch(torch.autograd.Function):
    """batch_sparse_tensor (utils.py:659-670) of M subnets: (features [M, L, C], int32 coordinates [M, L, 4], keep_pad
    bool [M, L] or an empty tensor); the backward hands every subnet its rows of the gradient."""

    @staticmethod
    def forward(ctx, want_keep, coords, *feats):
        M, L, C_ = len(feats), max(f.shape[0] for f in feats), feats[0].shape[1]
        dev = feats[0].device
        feats = [f.contiguous() for f in feats]
        out = torch.empty(M, L, C_, dtype=torch.float32, device=dev)
        out_c = torch.empty(M, L, 4, dtype=torch.int32, device=dev)
        keep = torch.empty(M, L, dtype=torch.bool, device=dev) if want_keep else torch.empty(0, device=dev)
        call("pasco_mimo_batch", _ptrs(feats), _ptrs(coords), (C.c_int64 * M)(*[f.shape[0] for f in feats]), M, L, C_,
             ptr(out), ptr(out_c), ptr(keep) if want_keep else None)
        ctx.lens = [f.shape[0] for f in feats]
        ctx.mark_non_differentiable(out_c, keep)
        return out, out_c, keep

    @staticmethod
    def backward(ctx, g, _c, _k):
        return (None, None) + tuple(g[m, :n] for m, n in enumerate(ctx.lens))


def mimo_batch(feats: List[torch.Tensor], coords: List[torch.Tensor], keep_pad: bool = False):
    """The M (<= 8) subnets' fp32 rows [L_m, C] and int32 coordinates [L_m, 4] zero-padded to L = max L_m in one launch:
    (features [M, L, C], coordinates [M, L, 4], keep_pad bool [M, L] or None) with keep_pad = any feature or coordinate
    != 0, the reference's rule (decoder_v3.py:443-446), not "row < L_m"."""
    out, out_c, keep = MimoBatch.apply(keep_pad, tuple(_i32(c).contiguous() for c in coords), *[f.float() for f in feats])
    return out, out_c, keep if keep_pad else None


# ----------------------------------------------------------------------------------------------
# fused BatchNorm (+ activation) over rows
# ----------------------------------------------------------------------------------------------
def column_stats(x: torch.Tensor) -> torch.Tensor:
    """float64 [2, C]: column sums and sums of squares."""
    stats = torch.zeros(2, x.shape[1], dtype=torch.float64, device=x.device)
    call("pasco_bn_stats", ptr(x), x.shape[0], x.shape[1], ptr(stats))
    return stats


def affine_act(x, scale, shift, act: int = 0, residual=None):
    y = torch.empty_like(x)
    call("pasco_affine_act", ptr(x), x.shape[0], x.shape[1], ptr(scale), ptr(shift), act, ptr(residual), ptr(y))
    return y


def _bn_forward_coefs(x, gamma, beta, eps, group, running_mean, running_var, momentum):
    """Training-mode BatchNorm coefficients of x [N, C]: column statistics (left by the producing convolution's epilogue
    when available, else one reduction pass; summed over `group` for SyncBatchNorm) → one coefficient kernel that also
    updates the running statistics.  Returns scale, shift (y = x*scale + shift), mean, rstd, count_dev."""
    n, c = x.shape
    dev = x.device
    stats = take_pending_stats(x)
    if stats is None:
        stats = column_stats(x)
    count_dev = None
    if group is not None:
        packed = torch.cat([stats.view(-1), torch.full((1,), float(n), dtype=torch.float64, device=dev)])
        torch.distributed.all_reduce(packed, group=group)
        stats, count_dev = packed[:-1].contiguous(), packed[-1:].contiguous()
    scale, shift, mean, rstd = (torch.empty(c, dtype=torch.float32, device=dev) for _ in range(4))
    call("pasco_bn_finalize", ptr(stats), ptr(count_dev), C.c_double(float(n)), c, ptr(gamma), ptr(beta), C.c_float(eps),
         C.c_float(momentum if momentum is not None else 0.1), ptr(scale), ptr(shift), ptr(mean), ptr(rstd),
         ptr(running_mean), ptr(running_var))
    return scale, shift, mean, rstd, count_dev


def _bn_backward(gy, x, gamma, scale, shift, mean, rstd, count_dev, act, group, n):
    """Gradient of y = act(BN(x)) w.r.t. x, gamma, beta: one reduce pass → one coefficient kernel → one apply pass."""
    gy = gy.contiguous()
    c = x.shape[1]
    dev = x.device
    sums = torch.zeros(2, c, dtype=torch.float64, device=dev)
    call("pasco_bn_bwd_reduce", ptr(gy), ptr(x), x.shape[0], c, ptr(scale), ptr(shift), act, ptr(sums))
    div = 1.0
    if group is not None:
        # sums are global after the all-reduce; every rank then holds the global dgamma/dbeta, and the gradient
        # all-reduce (mean over ranks) of the data-parallel step leaves them unchanged only if divided here
        torch.distributed.all_reduce(sums, group=group)
        div = float(torch.distributed.get_world_size(group))
    ca, cb, cc, gg, gb = (torch.empty(c, dtype=torch.float32, device=dev) for _ in range(5))
    call("pasco_bn_bwd_coefs", ptr(sums), ptr(count_dev), C.c_double(float(n)), c, ptr(gamma), ptr(mean), ptr(rstd),
         C.c_float(div), ptr(ca), ptr(cb), ptr(cc), ptr(gg), ptr(gb))
    gx = torch.empty_like(x)
    call("pasco_bn_bwd_apply", ptr(gy), ptr(x), x.shape[0], c, ptr(scale), ptr(shift), act,
         ptr(ca), ptr(cb), ptr(cc), ptr(gx))
    return gx, gg, gb


class BatchNormAct(torch.autograd.Function):
    """y = act(BN(x)) with training-mode batch statistics over all rows (optionally summed over ranks =
    SyncBatchNorm).  Forward: column sums → one coefficient kernel (scale/shift, mean/rstd, running statistics) →
    one apply pass; backward: one reduce pass → one coefficient kernel → one apply pass."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps, act, group, running_mean=None, running_var=None, momentum=0.1):
        x = x.contiguous()
        scale, shift, mean, rstd, count_dev = _bn_forward_coefs(x, gamma, beta, eps, group, running_mean, running_var, momentum)
        y = affine_act(x, scale, shift, act)
        ctx.save_for_backward(x, gamma, scale, shift, mean, rstd, count_dev)
        ctx.act, ctx.group, ctx.n = act, group, x.shape[0]
        return y

    @staticmethod
    def backward(ctx, gy):
        x, gamma, scale, shift, mean, rstd, count_dev = ctx.saved_tensors
        gx, gg, gb = _bn_backward(gy, x, gamma, scale, shift, mean, rstd, count_dev, ctx.act, ctx.group, ctx.n)
        return gx, gg, gb, None, None, None, None, None, None


class BNActConv(torch.autograd.Function):
    """out = SparseConv(act(BN(x)))  as ONE autograd node on the plane-gather path: the BatchNorm apply pass writes the
    normalised activations directly as bf16 planes (hi [+ lo]) — the only form the convolution and its weight gradient
    read — so the fp32 copy of act(BN(x)) never exists: same HBM bytes as the plain apply pass, no separate split pass,
    and the planes double as the saved tensor of the backward pass (pre-activation residual blocks, mink.py:618-658:
    BN → ReLU → conv, twice per block)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, weight, bias, eps, act, group, running_mean, running_var, momentum, kmap, packs):
        x = x.contiguous()
        scale, shift, mean, rstd, count_dev = _bn_forward_coefs(x, gamma, beta, eps, group, running_mean, running_var, momentum)
        hi, lo = split_planes(x, scale, shift, act)
        out = conv_apply(x, weight, kmap.nbr, kmap.n_out, False, None, bias.view(-1).contiguous() if bias is not None else None,
                         packs=packs, want_stats=True, planes=(hi, lo))
        ctx.kmap, ctx.packs, ctx.has_bias = kmap, packs, bias is not None
        ctx.act, ctx.group, ctx.n, ctx.has_lo = act, group, x.shape[0], lo is not None
        ctx.save_for_backward(x, gamma, scale, shift, mean, rstd, count_dev, weight, hi, *([lo] if lo is not None else []))
        return out

    @staticmethod
    def backward(ctx, g):
        x, gamma, scale, shift, mean, rstd, count_dev, weight, hi = ctx.saved_tensors[:9]
        lo = ctx.saved_tensors[9] if ctx.has_lo else None
        kmap = ctx.kmap
        g = g.contiguous()
        K, Cin, Cout = weight.shape
        g_planes = split_planes(g)
        nbr_t, koff_t = kmap.transposed()
        gy = conv_apply(g, weight, nbr_t, kmap.n_in, True, koff_t, packs=ctx.packs, planes=g_planes)
        gw = conv_wgrad(x, g, kmap.nbr, K, Cin, Cout, in_planes=(hi, lo), g_planes=g_planes) if ctx.needs_input_grad[3] else None
        gb = g.sum(0, keepdim=True) if ctx.has_bias and ctx.needs_input_grad[4] else None
        gx, gg, gbeta = _bn_backward(gy, x, gamma, scale, shift, mean, rstd, count_dev, ctx.act, ctx.group, ctx.n)
        return gx, gg, gbeta, gw, gb, None, None, None, None, None, None, None, None


def inference_fusion(flag: bool) -> None:
    global _INFER_FUSION
    _INFER_FUSION = bool(flag)


def inference_fusion_active(module) -> bool:
    """True when `module` (a BatchNorm or a network) runs in eval mode with gradients disabled and the inference fusions
    are on: nothing is recorded for a backward pass, so a BatchNorm with running statistics is a per-channel affine that
    can be folded into the planes a convolution gathers and into the epilogue of the convolution before it.  With
    gradients enabled, eval mode keeps its differentiable path (frozen-BatchNorm fine-tuning)."""
    return _INFER_FUSION and not module.training and not torch.is_grad_enabled()


def bn_eval_coefs(bn) -> Tuple[torch.Tensor, torch.Tensor]:
    """(scale, shift) of an eval-mode BatchNorm from its running statistics: BN(x) = x*scale + shift.  The one place these
    coefficients are computed (batchnorm_rows, bn_act_conv and the inference epilogue all use it)."""
    w = bn.weight if bn.weight is not None else 1.0
    scale = w * torch.rsqrt(bn.running_var + bn.eps)
    shift = (bn.bias if bn.bias is not None else 0.0) - bn.running_mean * scale
    return scale, shift


def bn_act_conv_route(bn, x, weight, kmap: "KernelMap") -> str:
    """How bn_act_conv runs conv(act(BatchNorm(x))): 'fused' (training, BNActConv: the BatchNorm apply pass writes the
    planes the convolution gathers), 'eval_split' (eval mode without gradients: one split_planes pass applies the
    running-statistics affine + activation and writes the planes; no autograd node) or 'unfused' (batchnorm_rows, then
    SparseConv).  The fused forms need the plane-gather tensor-core path."""
    K, Cin, Cout = weight.shape
    if bn.running_mean is None or not x.is_cuda:
        return "unfused"
    if bn.training:
        ok = (conv_path("fwd", Cin, Cout, kmap.K, kmap.nbr, kmap.n_out) == "planes"
              and conv_path("dgrad", Cout, Cin, kmap.K, kmap.nbr, kmap.n_in) == "planes"
              and conv_path("wgrad", Cin, Cout, kmap.K, kmap.nbr, kmap.n_out) == "planes")
        return "fused" if ok else "unfused"
    if inference_fusion_active(bn) and conv_path("fwd", Cin, Cout, kmap.K, kmap.nbr, kmap.n_out) == "planes":
        return "eval_split"
    return "unfused"


def bn_act_conv(bn, x: torch.Tensor, act: int, group, weight, bias, kmap: "KernelMap", packs=None) -> torch.Tensor:
    """conv(act(BatchNorm(x))) — fused (BNActConv) when the layer runs on the plane-gather tensor-core path in training
    mode, one split pass + the convolution in eval mode without gradients, the two separate nodes otherwise
    (bn_act_conv_route)."""
    route = bn_act_conv_route(bn, x, weight, kmap)
    if route == "eval_split":
        scale, shift = bn_eval_coefs(bn)
        planes = split_planes(x.contiguous(), scale.contiguous(), shift.contiguous(), act)
        return conv_apply(x, weight, kmap.nbr, kmap.n_out, False, None, bias.view(-1).contiguous() if bias is not None else None,
                          packs=packs, planes=planes)
    if route == "unfused":
        return SparseConv.apply(batchnorm_rows(bn, x, act, group), weight, bias, kmap, packs)
    with torch.no_grad():
        bn.num_batches_tracked += 1
    mom = bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked)
    return BNActConv.apply(x, bn.weight, bn.bias, weight, bias, bn.eps, act, group, bn.running_mean, bn.running_var, mom,
                           kmap, packs)


ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2


def _act_torch(z: torch.Tensor, act: int) -> torch.Tensor:
    if act == ACT_RELU:
        return torch.relu(z)
    if act == ACT_LEAKY:
        return torch.nn.functional.leaky_relu(z, 0.01)
    return z


def batchnorm_rows(bn, x: torch.Tensor, act: int = ACT_NONE, group=None) -> torch.Tensor:
    """act(BatchNorm(x)) over the rows of x [N, C] with the parameters / running statistics of a torch
    BatchNorm1d/3d/SyncBatchNorm module `bn`.  Training (or no running statistics): batch statistics through the fused
    kernels (ops.BatchNormAct).  Eval: a per-channel affine — through one fused kernel when no gradient is needed, through
    differentiable torch ops otherwise (frozen-BN fine-tuning keeps its graph)."""
    use_batch_stats = bn.training or bn.running_mean is None
    if use_batch_stats:
        if bn.training and bn.num_batches_tracked is not None:
            with torch.no_grad():
                bn.num_batches_tracked += 1
        gamma = bn.weight if bn.weight is not None else torch.ones(x.shape[1], device=x.device)
        beta = bn.bias if bn.bias is not None else torch.zeros(x.shape[1], device=x.device)
        mom = bn.momentum
        if mom is None and bn.num_batches_tracked is not None:          # cumulative moving average
            mom = 1.0 / float(bn.num_batches_tracked)
        rm, rv = (bn.running_mean, bn.running_var) if bn.training else (None, None)
        return BatchNormAct.apply(x, gamma, beta, bn.eps, act, group, rm, rv, mom)
    scale, shift = bn_eval_coefs(bn)
    if torch.is_grad_enabled() and (x.requires_grad or scale.requires_grad or shift.requires_grad):
        return _act_torch(x * scale + shift, act)
    return affine_act(x.contiguous(), scale.contiguous(), shift.contiguous(), act)


# ----------------------------------------------------------------------------------------------
# masked cross-attention of a few queries over all voxels (MaskPLS decoder)
# ----------------------------------------------------------------------------------------------
def pack_mask_bits(mask: torch.Tensor) -> torch.Tensor:
    """bool [Q,P] (True = masked) → int32 bit rows [Q, 2*ceil(P/64)], keys beyond P masked."""
    Q, P = mask.shape
    W = 2 * ((P + 63) // 64)
    pad = W * 32 - P
    m = torch.nn.functional.pad(mask, (0, pad), value=True) if pad else mask
    sh = torch.arange(32, device=mask.device, dtype=torch.int64)
    words = (m.view(Q, W, 32).to(torch.int64) << sh).sum(-1)
    return words.to(torch.int32).contiguous()


def attention_mask_bits(logits: torch.Tensor, key_parent: torch.Tensor, rows: Optional[torch.Tensor] = None,
                        parent_of: Optional[torch.Tensor] = None, n_parent: Optional[int] = None) -> torch.Tensor:
    """The attention mask of transformer_predictor_v2.py:220-289 and 164 as pack_mask_bits' int32 [Q, 2*ceil(P/64)]
    bit rows, without a [Q, P] intermediate: key v is masked for query q unless a scale-1 voxel u of v's stride-s block
    has logits[rows[u], q] > 0; a query with every key masked attends to all P keys.
    logits [*, Q] float32 with unit column stride (a column slice is fine); rows [n] int32 = the logit row of each
    scale-1 voxel (None: voxel u is row u); parent_of [n] int32 = each voxel's row among the n_parent stride-s voxels
    (None: s = 1); key_parent [P] int32 = each key's row among those (−1: no voxel, masked)."""
    assert logits.dtype == torch.float32 and logits.is_cuda and logits.dim() == 2 and logits.stride(1) == 1
    Q = logits.shape[1]
    n_child = rows.shape[0] if rows is not None else logits.shape[0]
    if parent_of is None:
        n_parent = n_child
    P = key_parent.shape[0]
    dev = logits.device
    pooled = torch.zeros(n_parent, (Q + 31) // 32, dtype=torch.int32, device=dev)
    seen = torch.zeros(Q, dtype=torch.int32, device=dev)
    bits = torch.empty(Q, 2 * ((P + 63) // 64), dtype=torch.int32, device=dev)
    call("pasco_attn_mask_bits", logits.data_ptr(), logits.stride(0), Q, ptr(rows), n_child, ptr(parent_of), n_parent,
         ptr(key_parent), P, ptr(pooled), ptr(seen), ptr(bits))
    return bits


class MaskedCrossAttention(torch.autograd.Function):
    """out[q] = concat_h softmax_v(scale·q_h·k_h[v] | mask[q,v]) · v_h[v]  — blocks.py:73-92 with the mask of
    transformer_predictor_v2.py:220-289.  q [Q, H*D] with any Q >= 1, k / v [P, H*D], D <= 64 and a multiple of 4,
    mask = int32 bit rows [Q, 2*ceil(P/64)] (attention_mask_bits, pack_mask_bits), bool [Q, P] (True = masked) or
    None.  Forward: two streaming wgmma passes (row statistics, then output); backward: one streaming pass with five wgmma GEMMs per 64-key tile that recomputes the probabilities from the
    saved log-sum-exp (xattn.cu).  Each pass splits the keys into chunks whose shares of out / dq are added in a fixed
    order; the per-chunk scratch comes from the library's own stream-ordered pool.  The kernels hold 128 queries at a
    time: above 128 every block of 128 queries streams K and V again, and the backward adds the blocks' dk / dv
    partials in block order (a workspace of (ceil(Q/128) - 1) * 2 * P * H*D floats), so results stay run-to-run
    identical."""

    @staticmethod
    def forward(ctx, q, k, v, mask, heads: int):
        q, k, v = q.contiguous().float(), k.contiguous().float(), v.contiguous().float()
        Q, HD = q.shape
        P = k.shape[0]
        D = HD // heads
        scale = float(D) ** -0.5
        bits = pack_mask_bits(mask) if mask is not None and mask.dtype == torch.bool else mask
        out = torch.zeros(Q, HD, dtype=torch.float32, device=q.device)
        lse = torch.empty(heads, Q, dtype=torch.float32, device=q.device)
        call("pasco_xattn_forward", ptr(q), ptr(k), ptr(v), ptr(bits), Q, P, heads, D, C.c_float(scale), ptr(out),
             ptr(lse))
        ctx.save_for_backward(q, k, v, bits, out, lse)
        ctx.heads, ctx.scale = heads, scale
        return out

    @staticmethod
    def backward(ctx, go):
        q, k, v, bits, out, lse = ctx.saved_tensors
        H, scale = ctx.heads, ctx.scale
        Q, HD = q.shape
        P = k.shape[0]
        go = go.contiguous().float()
        dq = torch.zeros_like(q)
        dk, dv = torch.empty_like(k), torch.empty_like(v)
        call("pasco_xattn_backward", ptr(q), ptr(k), ptr(v), ptr(bits), ptr(lse), ptr(out), ptr(go), Q, P, H, HD // H,
             C.c_float(scale), ptr(dq), ptr(dk), ptr(dv))
        return dq, dk, dv, None, None


def cross_attention(mha: torch.nn.MultiheadAttention, q: torch.Tensor, kv: torch.Tensor,
                    mask: Optional[torch.Tensor]) -> torch.Tensor:
    """`mha(q, kv, kv, attn_mask=mask)` of blocks.py:73-92 for one scene: q [Q, d] (query position already added),
    kv [P, d] (key position already added), mask = attention_mask_bits' bit rows, bool [Q, P] (True = masked) or None
    → [Q, d].  The K / V projections
    over all voxels run on the wgmma GEMM, the masked softmax·V on MaskedCrossAttention."""
    d = q.shape[-1]
    wq, wk, wv = mha.in_proj_weight.split(d, 0)
    bq, bk, bv = mha.in_proj_bias.split(d, 0)
    kv = kv.contiguous()
    o = MaskedCrossAttention.apply(torch.nn.functional.linear(q, wq, bq), linear(kv, wk, bk), linear(kv, wv, bv), mask,
                                   mha.num_heads)
    return mha.out_proj(o)


# ----------------------------------------------------------------------------------------------
# the mask transformer's sine position encoding (posenc.cu)
# ----------------------------------------------------------------------------------------------
SINE_SPAN = 64          # the encoding table covers coordinates [-SINE_SPAN, SINE_SPAN]; it is constant beyond |x| >= 32
_SINE_TABLES = {}


def sine_table(n: int, temperature, dev) -> torch.Tensor:
    """One axis of PositionEmbeddingSineSparse(n, temperature, normalize=True) (position_encoding.py:94-131) over the
    coordinates -SINE_SPAN .. SINE_SPAN, computed by the reference's own torch expression, so every value carries torch's
    bits: fp32 [2·SINE_SPAN + 1, n].  Cached per (n, temperature, device)."""
    key = (n, temperature, type(temperature), dev)
    t = _SINE_TABLES.get(key)
    if t is None:
        x = torch.arange(-SINE_SPAN, SINE_SPAN + 1, device=dev).float()
        x = x / (x + 1e-6) * (2 * math.pi)
        dim_t = torch.arange(n, dtype=torch.float, device=dev)
        dim_t = temperature ** (2 * (dim_t // 2) / n)
        p = x[:, None] / dim_t
        t = _SINE_TABLES[key] = torch.stack((p[:, 0::2].sin(), p[:, 1::2].cos()), dim=1).flatten(1).contiguous()
    return t


def sine_pos(coords: torch.Tensor, n: int, out: Optional[torch.Tensor] = None, add: bool = False,
             temperature=10000) -> torch.Tensor:
    """PositionEmbeddingSineSparse(n, normalize=True) of integer coordinates, bit for bit: coords int32 / int64 [P, 4]
    (b, x, y, z) or [P, 3] (x, y, z), any row pitch → fp32 [P, 3n].  add=False writes the encoding (into `out` when given,
    else a new tensor); add=True adds it into `out` in place, one read-modify-write.  `out` may be a column slice: unit
    column stride, any row pitch.  n even, 2 <= n <= 256."""
    assert coords.is_cuda and coords.dtype in (torch.int32, torch.int64) and coords.dim() == 2
    assert coords.shape[1] in (3, 4), "sine_pos: coordinates are [P, 4] (b, x, y, z) or [P, 3]"
    P = coords.shape[0]
    if coords.stride(1) != 1 or (P > 1 and coords.stride(0) < coords.shape[1]):
        coords = coords.contiguous()
    if out is None:
        assert not add, "sine_pos: add=True adds into `out`"
        out = torch.empty(P, 3 * n, dtype=torch.float32, device=coords.device)
    assert out.dtype == torch.float32 and out.device == coords.device and tuple(out.shape) == (P, 3 * n)
    assert out.stride(1) == 1 and (P <= 1 or out.stride(0) >= 3 * n), "sine_pos: out needs unit column stride"
    table = sine_table(n, temperature, coords.device)
    call("pasco_sine_pos", C.c_void_p(coords.data_ptr() + coords.element_size() * (coords.shape[1] - 3)),
         int(coords.dtype == torch.int64), P, coords.stride(0) if P > 1 else coords.shape[1], ptr(table), -SINE_SPAN,
         table.shape[0], n, C.c_void_p(out.data_ptr()), out.stride(0) if P > 1 else 3 * n, int(add))
    return out


class AddSinePos(torch.autograd.Function):
    """y + sine_pos(coords, n), added into y's rows in place; the gradient with respect to y is the identity."""

    @staticmethod
    def forward(ctx, y, coords, n):
        ctx.mark_dirty(y)
        return sine_pos(coords, n, out=y, add=True)

    @staticmethod
    def backward(ctx, g):
        return g, None, None


def add_sine_pos(y: torch.Tensor, coords: torch.Tensor, n: int) -> torch.Tensor:
    """y += PositionEmbeddingSineSparse(n, normalize=True)(coords) in place, autograd-transparent (y must be a tensor no
    backward pass reads, such as a fresh Linear output).  Returns y."""
    return AddSinePos.apply(y, coords, n)


# ----------------------------------------------------------------------------------------------
# dense Linear layers on the tensor-core conv kernel (K = 1, identity rows, column chunks <= 256)
# ----------------------------------------------------------------------------------------------
def _data_ptr_at(t: torch.Tensor, col: int) -> int:
    return t.data_ptr() + 4 * col


def _linear_tc_ok(n_rows: int, cin: int, cout: int) -> bool:
    return (not _FORCE_SIMT) and n_rows >= 4096 and cin % 64 == 0 and cout % 64 == 0


def _gemm_rows(x: torch.Tensor, w_nk: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor) -> None:
    """out[:, :] = x @ w_nkᵀ (+ bias) with w_nk [N, K] row-major (torch Linear layout), N in chunks of <= 256 columns."""
    global _PENDING_STATS
    _PENDING_STATS = None
    n_rows, kdim = x.shape
    N = w_nk.shape[0]
    assert x.is_contiguous() and out.is_contiguous() and kdim % 64 == 0 and N % 16 == 0
    for c0 in range(0, N, 256):
        cw = min(256, N - c0)
        wchunk = w_nk[c0:c0 + cw].contiguous()                       # [cw, K]  == ME layout [1, Cin'=cw, Cout'=K]
        packed = PackedWeights().get(wchunk.view(1, cw, kdim), True)  # B[n][k] = w[n][k]
        b = bias[c0:c0 + cw].contiguous() if bias is not None else None
        call("pasco_conv_forward_tc", ptr(x), n_rows, None, 1, n_rows, kdim, cw, ptr(packed), None, ptr(b), None,
             C.c_void_p(_data_ptr_at(out, c0)), _PRECISION, 0, N)


class LinearTC(torch.autograd.Function):
    """y = x @ Wᵀ + b for tall x [N, Cin] on the wgmma conv kernel (bf16x3 / bf16 like the convolutions) instead of
    an fp32 CUDA-core library GEMM.  W is [Cout, Cin] (torch Linear layout)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        x = x.contiguous().float()
        y = torch.empty(x.shape[0], weight.shape[0], dtype=torch.float32, device=x.device)
        _gemm_rows(x, weight.detach(), bias.detach() if bias is not None else None, y)
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        gy = gy.contiguous().float()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = torch.empty_like(x)
            _gemm_rows(gy, weight.detach().t().contiguous(), None, gx)          # gx = gy @ W
        if ctx.needs_input_grad[1]:
            cout, cin = weight.shape
            gw = torch.empty(cout, cin, dtype=torch.float32, device=x.device)
            for c0 in range(0, cin, 256):                                        # dW[:, c0:c0+cw] = gyᵀ @ x[:, c0:c0+cw]
                cw = min(256, cin - c0)
                dw = torch.zeros(1, cout, cw, dtype=torch.float32, device=x.device)
                call("pasco_conv_wgrad_tc", ptr(gy), gy.shape[0], None, 1, gy.shape[0], cout, cw,
                     C.c_void_p(_data_ptr_at(x, c0)), ptr(dw), _PRECISION, 0, cin)
                gw[:, c0:c0 + cw] = dw[0]
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = gy.sum(0)
        return gx, gw, gb


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.linear for [N, Cin] inputs: tensor-core path when the shape allows (N >= 4096, Cin, Cout multiples of 64),
    the fp32 library GEMM otherwise (exactly what MinkowskiEngine does for 1x1 convolutions)."""
    if x.is_cuda and x.ndim == 2 and _linear_tc_ok(x.shape[0], weight.shape[1], weight.shape[0]):
        return LinearTC.apply(x, weight, bias)
    return torch.nn.functional.linear(x, weight, bias)


# ----------------------------------------------------------------------------------------------
# test-time post-processing (panoptic.cu): M-subnet ensemble and panoptic inference on sparse rows of the reference grid
# ----------------------------------------------------------------------------------------------
def plane_cols(q: int) -> int:
    """Columns of the bf16 planes of a [N, q] mask matrix: q rounded up to the tensor-core channel rule (16)."""
    return (q + 15) // 16 * 16


def pose_lookup(table: HashTable, T: torch.Tensor, size: Sequence[int]) -> Tuple[torch.Tensor, torch.Tensor]:
    """Every cell of the reference grid `size` → the row of `table` (keys with batch index 0) at the cell's nearest
    voxel under the pose T (transform_utils.transform): (cell_row int32 [cells], −1 = none; cell_row >= 0 as uint8)."""
    cells = int(size[0]) * int(size[1]) * int(size[2])
    dev = table.keys.device
    cell_row = torch.empty(cells, dtype=torch.int32, device=dev)
    mask = torch.empty(cells, dtype=torch.uint8, device=dev)
    t = T.detach().to("cpu", torch.float32).reshape(4, 4)[:3].contiguous().view(-1).tolist()
    call("pasco_pose_lookup", ptr(table.keys), ptr(table.vals), table.capacity, (C.c_float * 12)(*t), int(size[0]),
         int(size[1]), int(size[2]), ptr(cell_row), ptr(mask))
    return cell_row, mask


def cell_mask_or(cell_row: torch.Tensor, mask: torch.Tensor) -> None:
    call("pasco_cell_mask_or", ptr(cell_row), cell_row.shape[0], ptr(mask))


def lookup_rows(cell_row: torch.Tensor, lin: torch.Tensor) -> torch.Tensor:
    out = torch.empty(lin.shape[0], dtype=torch.int32, device=lin.device)
    call("pasco_lookup_rows", ptr(cell_row), ptr(lin), lin.shape[0], ptr(out))
    return out


def box_cells(coords: torch.Tensor, lo: Sequence[int], hi: Sequence[int], size: Sequence[int], counts: torch.Tensor):
    """The rows of coords ([N, 4] (b, x, y, z), b ignored) with lo <= (x, y, z) <= hi at cells (x, y, z) − lo of the box
    `size` → (cell_row int32 [cells], −1 = none; cell_row >= 0 as uint8).  counts (int32 [2] on the device, zeroed)
    receives the number of rows outside [lo, hi] and of rows at a cell another row already holds; nothing is read back."""
    X, Y, Z = (int(s) for s in size)
    dev = coords.device
    c = coords if coords.dtype == torch.int32 and coords.is_contiguous() else coords.to(torch.int32).contiguous()
    if c.dim() != 2 or c.shape[1] != 4:
        raise ValueError(f"box_cells: coordinates must be [N, 4], got {tuple(coords.shape)}")
    cell_row = torch.full((X * Y * Z,), -1, dtype=torch.int32, device=dev)
    mask = torch.zeros(X * Y * Z, dtype=torch.uint8, device=dev)
    call("pasco_box_cells", ptr(c), c.shape[0], int_array(lo), int_array(hi), X, Y, Z, ptr(cell_row), ptr(mask),
         ptr(counts))
    return cell_row, mask


def _mask_outputs(n: int, q: int, dev, planes: bool, colsum: bool):
    qp = plane_cols(q)
    out = torch.empty(n, q, dtype=torch.float32, device=dev)
    hi = torch.empty(n, qp, dtype=torch.bfloat16, device=dev) if planes else None
    lo = torch.empty(n, qp, dtype=torch.bfloat16, device=dev) if planes else None
    cs = torch.empty(q, dtype=torch.float32, device=dev) if colsum else None
    nz = torch.empty(n, dtype=torch.uint8, device=dev)
    return out, hi, lo, qp, cs, nz


def mask_rows_sigmoid(logits: torch.Tensor, rows: torch.Tensor, planes: bool = True):
    """sigmoid(logits[rows]) → (probs fp32 [n, Q], (hi, lo) bf16 planes [n, plane_cols(Q)] or None, column sums [Q] or
    None, non-zero row flags uint8 [n])."""
    logits = logits.detach().float().contiguous()
    out, hi, lo, qp, cs, nz = _mask_outputs(rows.shape[0], logits.shape[1], logits.device, planes, planes)
    call("pasco_mask_rows_sigmoid", ptr(logits), ptr(rows), rows.shape[0], logits.shape[1], ptr(out), ptr(hi), ptr(lo),
         qp, ptr(cs), ptr(nz))
    return out, ((hi, lo) if planes else None), cs, nz


def mask_merge(a: torch.Tensor, cell_a: torch.Tensor, b: Optional[torch.Tensor], cell_b: Optional[torch.Tensor],
               lin: torch.Tensor, a_col: torch.Tensor, b_col: Optional[torch.Tensor], weight: int,
               gate: Optional[torch.Tensor] = None, planes: bool = True):
    """Rows at the cells lin: column j = (a[:, a_col[j]]·weight + b[:, b_col[j]]) / (weight + 1) (a missing row is a
    zero row), times gate[cell] when given.  Returns what mask_rows_sigmoid returns."""
    q = a_col.shape[0]
    out, hi, lo, qp, cs, nz = _mask_outputs(lin.shape[0], q, a.device, planes, planes)
    call("pasco_mask_merge", ptr(a), ptr(cell_a), a.shape[1], ptr(b), ptr(cell_b), b.shape[1] if b is not None else 0,
         ptr(lin), lin.shape[0], ptr(a_col), ptr(b_col), q, int(weight), ptr(gate), ptr(out), ptr(hi), ptr(lo), qp, ptr(cs),
         ptr(nz))
    return out, ((hi, lo) if planes else None), cs, nz


def softmax_rows(logits: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    logits = logits.detach().float().contiguous()
    out = torch.empty(rows.shape[0], logits.shape[1], dtype=torch.float32, device=logits.device)
    call("pasco_softmax_rows", ptr(logits), ptr(rows), rows.shape[0], logits.shape[1], ptr(out))
    return out


def soft_iou(a_prob, a_planes, a_sum, b_prob, b_planes, b_sum, nbr: torch.Tensor, threshold: float) -> torch.Tensor:
    """Gated soft IoU [Q, Q] between the mask sets A (rows of the anchor) and B; nbr int32 [N_b] = the anchor row at the
    cell of every row of B (−1 none).  The intersections are the weight gradient of a K = 1 convolution from A's planes
    to B's (bf16x3, fixed-order reduction); a width outside the tensor-core channel rule takes the CUDA-core kernel."""
    q = a_prob.shape[1]
    dev = a_prob.device
    nb = b_prob.shape[0]
    nbr = nbr.view(1, -1)
    qp = plane_cols(q)
    # conv_path only decides tensor cores vs CUDA cores here: with K = 1 it names the register-gather kernel, but the
    # masks already exist as planes, so every tensor-core case takes the plane-gather weight gradient
    if conv_path("wgrad", qp, qp, 1, nbr, nb) == "simt":
        inter = torch.zeros(1, q, q, dtype=torch.float32, device=dev)
        pitch = q
        if nb:
            call("pasco_conv_wgrad_simt", ptr(a_prob), ptr(nbr), 1, nb, q, q, ptr(b_prob), ptr(inter))
    else:
        inter = torch.zeros(1, qp, qp, dtype=torch.float32, device=dev)
        pitch = qp
        if nb:
            (ah, al), (bh, bl) = a_planes, b_planes
            call("pasco_conv_wgrad_planes", ptr(ah), ptr(al), a_prob.shape[0], ptr(nbr), 1, nb, qp, qp, ptr(bh), ptr(bl),
                 ptr(inter), 3, 0, 0)
    gated = torch.empty(q, q, dtype=torch.float32, device=dev)
    call("pasco_soft_iou", ptr(inter), q, pitch, ptr(a_sum), ptr(b_sum), float(threshold), ptr(gated))
    return gated


def sem_ensemble(probs: List[torch.Tensor], cell_rows: List[torch.Tensor], lin: torch.Tensor,
                 gate: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Mean class distribution over the subnets at the cells lin (absent subnet = one-hot class 0) → (argmax int32,
    max fp32); gate (uint8 [cells], zeroed) receives argmax != 0 at those cells."""
    n, K, M = lin.shape[0], probs[0].shape[1], len(probs)
    pred = torch.empty(n, dtype=torch.int32, device=lin.device)
    conf = torch.empty(n, dtype=torch.float32, device=lin.device)
    call("pasco_sem_ensemble", M, (C.c_void_p * M)(*[ptr(p) for p in probs]), (C.c_void_p * M)(*[ptr(c) for c in cell_rows]),
         ptr(lin), n, K, ptr(pred), ptr(conf), ptr(gate))
    return pred, conf


def _panoptic_passes(probs, qp, overlap_threshold, object_mask_threshold, thing_ids, vox_occ_threshold, dense: bool):
    """Passes 1, segments and 2 → (panoptic, semantic, confidence rows, device int32 [1 + 4Q (+ 1 + Q)] = the records
    (then the kept-query count and list when dense), win, m_win, c_sum or None)."""
    n, q = probs.shape
    K1 = qp.shape[1]
    dev = probs.device
    win = torch.empty(n, dtype=torch.int32, device=dev)
    m_win = torch.empty(n, dtype=torch.float32, device=dev)
    m_sum = torch.empty(n, dtype=torch.float32, device=dev)
    c_sum = torch.empty(n, dtype=torch.float32, device=dev) if dense else None
    areas = torch.zeros(2 * max(q, 1), dtype=torch.int32, device=dev)
    seg_of = torch.empty(max(q, 1), dtype=torch.int32, device=dev)
    cls_of = torch.empty(max(q, 1), dtype=torch.int32, device=dev)
    out = torch.zeros(1 + 4 * q + (1 + q if dense else 0), dtype=torch.int32, device=dev)
    pan = torch.empty(n, dtype=torch.int32, device=dev)
    sem = torch.empty(n, dtype=torch.int32, device=dev)
    conf = torch.empty(n, dtype=torch.float32, device=dev)
    if q == 0:
        return pan.zero_(), sem.zero_(), conf.zero_(), out, win, m_win, c_sum
    mask = 0
    for c in thing_ids:
        mask |= 1 << int(c)
    call("pasco_panoptic_pass1", ptr(probs.contiguous()), n, q, ptr(qp), K1, float(object_mask_threshold),
         float(vox_occ_threshold), ptr(win), ptr(m_win), ptr(m_sum), ptr(c_sum), ptr(areas))
    call("pasco_panoptic_segments", ptr(qp), q, K1, float(object_mask_threshold), float(overlap_threshold), mask,
         ptr(areas), ptr(seg_of), ptr(cls_of), ptr(out[:1 + 4 * q]), ptr(out[1 + 4 * q:]) if dense else None)
    call("pasco_panoptic_pass2", ptr(win), ptr(m_win), ptr(m_sum), n, ptr(seg_of), ptr(cls_of), ptr(pan), ptr(sem), ptr(conf))
    return pan, sem, conf, out, win, m_win, c_sum


def panoptic(probs: torch.Tensor, query_probs: torch.Tensor, overlap_threshold: float, object_mask_threshold: float,
             thing_ids: Sequence[int], vox_occ_threshold: float = 0.3):
    """helper.py:135-263 for one prediction: probs fp32 [N, Q] mask probabilities, query_probs fp32 [Q, K1].
    Returns (panoptic int32 [N], semantic int32 [N], confidence fp32 [N], records int32 [1 + 4Q] on the host)."""
    qp = query_probs.detach().float().contiguous()
    pan, sem, conf, records = _panoptic_passes(probs, qp, overlap_threshold, object_mask_threshold, thing_ids,
                                               vox_occ_threshold, False)[:4]
    return pan, sem, conf, records.cpu()


def panoptic_dense(probs: torch.Tensor, coords: torch.Tensor, query_probs: torch.Tensor, overlap_threshold: float,
                   object_mask_threshold: float, thing_ids: Sequence[int], min_c: Sequence[int], size: Sequence[int],
                   vox_occ_threshold: float = 0.3):
    """helper.py:135-281 for one prediction whose rows sit at coords int32 [N, 4] (batch 0): the passes of `panoptic`,
    then every dense volume panoptic_inference returns, channel-first over the box of `size` cells from min_c.
    Returns (panoptic rows int32 [N], records int32 [1 + 4Q] on the host, {"panoptic", "semantic" int32 [X, Y, Z],
    "confidence", "ins_uncertainty", "vox_uncertainty" fp32 [X, Y, Z], "all_mask_probs" fp32 [kq, X, Y, Z]}), or None
    when a row lies outside the box or in another batch (checked on a flag of its own, so a pending error of another
    pass is left to raise_pending_errors).  Two host synchronisations: the records, then the box check."""
    n, q = probs.shape
    dev = probs.device
    qp = query_probs.detach().float().contiguous()
    probs = probs.contiguous()
    pan, sem, conf, out, win, m_win, c_sum = _panoptic_passes(probs, qp, overlap_threshold, object_mask_threshold,
                                                              thing_ids, vox_occ_threshold, True)
    host = out.cpu()
    kq = int(host[1 + 4 * q])
    X, Y, Z = (int(s) for s in size)
    vol = {k: torch.zeros(X, Y, Z, dtype=dt, device=dev) for k, dt in
           (("panoptic", torch.int32), ("semantic", torch.int32), ("confidence", torch.float32),
            ("ins_uncertainty", torch.float32), ("vox_uncertainty", torch.float32))}
    vol["all_mask_probs"] = torch.zeros(kq, X, Y, Z, dtype=torch.float32, device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    call("pasco_panoptic_dense", ptr(coords), n, int_array(min_c), X, Y, Z, ptr(pan), ptr(sem), ptr(conf), ptr(win),
         ptr(m_win), ptr(c_sum), ptr(qp), qp.shape[1], ptr(probs), q, ptr(out[2 + 4 * q:2 + 4 * q + kq]), kq,
         ptr(vol["panoptic"]), ptr(vol["semantic"]), ptr(vol["confidence"]), ptr(vol["ins_uncertainty"]),
         ptr(vol["vox_uncertainty"]), ptr(vol["all_mask_probs"]) if kq else None, ptr(flag))
    if n and int(flag.item()):
        return pan, host[:1 + 4 * q], None
    return pan, host[:1 + 4 * q], vol


def sem_dense(probs: List[torch.Tensor], cell_rows: List[torch.Tensor], cells: int, subnets: bool = True,
              gate: Optional[torch.Tensor] = None) -> Tuple[Optional[List[torch.Tensor]], torch.Tensor]:
    """The dense class distributions fp32 [K, cells] of every subnet (when `subnets`; one-hot class 0 where a subnet has no
    row) and of their mean, as sem_ensemble computes it; gate (uint8 [cells]) receives the mean's argmax != 0."""
    M, K = len(probs), probs[0].shape[1]
    dev = probs[0].device
    subs = [torch.empty(K, cells, dtype=torch.float32, device=dev) for _ in range(M)] if subnets else None
    ens = torch.empty(K, cells, dtype=torch.float32, device=dev)
    call("pasco_sem_dense", M, (C.c_void_p * M)(*[ptr(p) for p in probs]), (C.c_void_p * M)(*[ptr(c) for c in cell_rows]),
         cells, K, (C.c_void_p * M)(*[ptr(s) for s in subs]) if subnets else None, ptr(ens), ptr(gate))
    return subs, ens


def class_gate(dense: torch.Tensor) -> torch.Tensor:
    """dense fp32 [K, X, Y, Z] → uint8 [X·Y·Z]: first argmax over the channels != 0."""
    d = dense.detach().float().contiguous()
    cells = d[0].numel()
    gate = torch.empty(cells, dtype=torch.uint8, device=d.device)
    call("pasco_class_gate", ptr(d), cells, d.shape[0], ptr(gate))
    return gate


# ----------------------------------------------------------------------------------------------
# evaluation passes (csrc/metrics.cu); the host finishing is pasco_b200/metrics.py
# ----------------------------------------------------------------------------------------------
CAL_BOUNDS = torch.linspace(0, 1, 16, dtype=torch.float32)     # torchmetrics' bins for n_bins = 15, in fp32


def _bounds():
    return (C.c_float * 16)(*CAL_BOUNDS.tolist())


def eval_gt(masks: torch.Tensor, seg_of_mask: torch.Tensor, label: torch.Tensor, G: int, K: int):
    """masks uint8 [n, cells], seg_of_mask int32 [n], label uint8 [cells] → (gt_id int32 [cells], counts int32 on the
    device: [n] mask sums, [G + 1] areas of the ids after unknown zeroing, [K + 1] known-cell class histogram)."""
    n, cells = masks.shape[0], label.numel()
    gt_id = torch.empty(cells, dtype=torch.int32, device=label.device)
    counts = torch.zeros(n + G + 1 + K + 1, dtype=torch.int32, device=label.device)
    call("pasco_eval_gt", ptr(masks), n, ptr(seg_of_mask), ptr(label), cells, G, K, ptr(gt_id), ptr(counts[:n]),
         ptr(counts[n:n + G + 1]), ptr(counts[n + G + 1:]))
    return gt_id, counts


def eval_pairs(lin: torch.Tensor, pan: torch.Tensor, gt_id: torch.Tensor, label: torch.Tensor, G: int, S: int,
               out: torch.Tensor) -> None:
    """out int32 [(G + 1)(S + 1) + S + 1], zeroed: the (gt id, pred id) intersections, then the predicted areas."""
    t = (G + 1) * (S + 1)
    call("pasco_eval_pairs", ptr(lin), ptr(pan), lin.shape[0], ptr(gt_id), ptr(label), label.numel(), G, S, ptr(out[:t]),
         ptr(out[t:]))


def eval_ssc(lin: torch.Tensor, pred: torch.Tensor, conf: torch.Tensor, label: torch.Tensor, K: int,
             sem_rows: Sequence, out: torch.Tensor) -> None:
    """out int32 [K*K + 64 + 1 + pad + 68], zeroed: the confusion counts, the calibration counts, the bad-row count and
    (8-byte aligned) the 34 double sums; sem_rows = [(softmax rows fp32 [n_m, K], cell map int32 [cells])] of the subnets
    averaged (may be empty)."""
    M = len(sem_rows)
    for p, c in sem_rows:
        if not (p.dtype == torch.float32 and p.dim() == 2 and p.shape[1] == K and p.device == label.device
                and p.is_contiguous() and c.dtype == torch.int32 and c.numel() == label.numel()
                and c.device == label.device and c.is_contiguous()):
            raise ValueError(f"eval_ssc: semantic rows must be fp32 [n, {K}] with an int32 cell map of {label.numel()} "
                             f"cells, got {p.dtype} {tuple(p.shape)} and {c.dtype} {tuple(c.shape)}")
    o = K * K + 65 + (K * K + 65) % 2
    sums = out[o:o + 68].view(torch.float64)
    call("pasco_eval_ssc", ptr(lin), ptr(pred), ptr(conf), lin.shape[0], ptr(label), label.numel(), K, _bounds(), M,
         (C.c_void_p * max(M, 1))(*[ptr(p) for p, _ in sem_rows]), (C.c_void_p * max(M, 1))(*[ptr(c) for _, c in sem_rows]),
         ptr(out[:K * K]), ptr(out[K * K:K * K + 64]), ptr(out[K * K + 64:K * K + 65]), ptr(sums))


def eval_vox(lin: torch.Tensor, pan: torch.Tensor, conf: torch.Tensor, gt_id: torch.Tensor, match: torch.Tensor,
             out: torch.Tensor) -> None:
    """out int32 [64], zeroed: [2][16] (count, correct) per slot, then the 16 double confidence sums."""
    call("pasco_eval_vox", ptr(lin), ptr(pan), ptr(conf), lin.shape[0], ptr(gt_id), gt_id.numel(), ptr(match),
         match.shape[0] - 1,
         _bounds(), ptr(out[:32]), ptr(out[32:].view(torch.float64)))


# dense forms (the volumes the reference's evaluate_all is given: row i = cell i)
def eval_gt_volume(gt_id: torch.Tensor) -> torch.Tensor:
    """gt_id int32 [cells] (eval_gt's) → fp32 [cells]: the gt_panoptic_seg volume evaluate_all returns."""
    out = torch.empty(gt_id.numel(), dtype=torch.float32, device=gt_id.device)
    call("pasco_eval_gt_volume", ptr(gt_id), gt_id.numel(), ptr(out))
    return out


def eval_pairs_dense(pan: torch.Tensor, gt_id: torch.Tensor, label: torch.Tensor, G: int, S: int,
                     out: torch.Tensor) -> None:
    """eval_pairs over a dense id volume pan int32 [cells]; out as eval_pairs'."""
    if not (pan.dtype == torch.int32 and pan.numel() == label.numel() and pan.device == label.device):
        raise ValueError(f"eval_pairs_dense: the id volume must be int32 of {label.numel()} cells on {label.device}, got "
                         f"{pan.dtype} {tuple(pan.shape)}")
    t = (G + 1) * (S + 1)
    call("pasco_eval_pairs_dense", ptr(pan), ptr(gt_id), ptr(label), label.numel(), G, S, ptr(out[:t]), ptr(out[t:]))


def eval_ssc_planes(prob: torch.Tensor, label: torch.Tensor, conf: Optional[torch.Tensor], out: torch.Tensor) -> torch.Tensor:
    """prob fp32 [K, cells] channel-major, label uint8 [cells], conf fp32 [cells] or None → the first-argmax volume int64
    [cells].  out int32 [K*K + 64 + 1 + pad + 68], zeroed, in eval_ssc's layout (confusion counts, calibration counts,
    bad-cell count, the 34 double sums); without conf only the confusion counts and the bad count are written."""
    K, cells = prob.shape[0], label.numel()
    if not (prob.dtype == torch.float32 and prob.dim() == 2 and prob.shape[1] == cells and prob.device == label.device):
        raise ValueError(f"eval_ssc_planes: class planes must be fp32 [K, {cells}] on {label.device}, got {prob.dtype} "
                         f"{tuple(prob.shape)}")
    if conf is not None and not (conf.dtype == torch.float32 and conf.numel() == cells and conf.device == label.device):
        raise ValueError(f"eval_ssc_planes: confidences must be fp32 [{cells}] on {label.device}, got {conf.dtype} "
                         f"{tuple(conf.shape)}")
    o = K * K + 65 + (K * K + 65) % 2
    pred = torch.empty(cells, dtype=torch.int64, device=label.device)
    call("pasco_eval_ssc_planes", ptr(prob), K, cells, ptr(label), ptr(conf), _bounds(), ptr(pred), ptr(out[:K * K]),
         ptr(out[K * K:K * K + 64]), ptr(out[K * K + 64:K * K + 65]), ptr(out[o:o + 68].view(torch.float64)))
    return pred


def eval_vox_dense(pan: torch.Tensor, conf: torch.Tensor, gt_id: torch.Tensor, match: torch.Tensor,
                   out: torch.Tensor) -> None:
    """eval_vox over dense volumes pan int32 / conf fp32 [cells]; out int32 [66], zeroed: [2][16] (count, correct) per
    slot, the 16 double confidence sums, then the count of counted cells with a confidence outside [0, 1]."""
    cells = gt_id.numel()
    if not (pan.dtype == torch.int32 and conf.dtype == torch.float32 and pan.numel() == conf.numel() == cells):
        raise ValueError(f"eval_vox_dense: the volumes must be int32 / fp32 of {cells} cells, got {pan.dtype} "
                         f"{tuple(pan.shape)} and {conf.dtype} {tuple(conf.shape)}")
    call("pasco_eval_vox_dense", ptr(pan), ptr(conf), ptr(gt_id), cells, ptr(match), match.shape[0] - 1, _bounds(),
         ptr(out[:32]), ptr(out[64:65]), ptr(out[32:64].view(torch.float64)))


# ------------------------------------------------------------------------------------------------
# training criterion of the reference's SetCriterion (csrc/setloss.cu)
# ------------------------------------------------------------------------------------------------
def setloss_sample(xyz: torch.Tensor, min_c: torch.Tensor, masks: torch.Tensor, unknown: torch.Tensor,
                   label: Optional[torch.Tensor], K: int):
    """xyz int32 [N, 4] (batch, x, y, z; rows of batch items other than 0 are left out), min_c int32 [3] (device), masks bool / uint8 [T, X, Y, Z], unknown bool [X, Y, Z], label
    uint8 [X, Y, Z] or None → (bits int32 [N, max(1, ⌈T/32⌉)], flags uint8 [N], lab int32 [N] or None, stats int32
    [T + 5]) in pasco_setloss_sample's layout."""
    T, size = masks.shape[0], tuple(unknown.shape)
    dev, N = xyz.device, xyz.shape[0]
    W = max(1, (T + 31) // 32)
    u8 = lambda t: (t.contiguous().view(torch.uint8) if t.dtype == torch.bool else t.to(torch.uint8).contiguous())  # noqa: E731
    m8 = u8(masks.reshape(T, -1)) if T else torch.zeros(1, dtype=torch.uint8, device=dev)
    bits = torch.empty(N, W, dtype=torch.int32, device=dev)
    flags = torch.empty(N, dtype=torch.uint8, device=dev)
    lab = torch.empty(N, dtype=torch.int32, device=dev) if label is not None else None
    stats = torch.zeros(T + 5, dtype=torch.int32, device=dev)
    call("pasco_setloss_sample", ptr(xyz), N, ptr(min_c), ptr(m8), T, ptr(u8(unknown)),
         ptr(u8(label) if label is not None else None), *size, K, ptr(bits), ptr(flags), ptr(lab), ptr(stats))
    return bits, flags, lab, stats


def match_cost(F: torch.Tensor, bits: torch.Tensor, T: int, flags: torch.Tensor, stats: torch.Tensor,
               query_logits: torch.Tensor, ids: torch.Tensor, class_weight: torch.Tensor, cost_mask: float,
               cost_class: float, cost_dice: float) -> torch.Tensor:
    """matcher_sparse.py:96-157 → C fp32 [Q, T].  F fp32 [N, Q]; query_logits fp32 [Q, K+1]; ids int32 [T]."""
    Q = F.shape[1]
    C_ = torch.empty(Q, T, dtype=torch.float32, device=F.device)
    call("pasco_setloss_match_cost", ptr(F), F.shape[0], Q, ptr(bits), T, ptr(flags), ptr(stats),
         ptr(query_logits), query_logits.shape[1], ptr(ids), ptr(class_weight), float(cost_mask), float(cost_class),
         float(cost_dice), ptr(C_))
    return C_


class PairSums(torch.autograd.Function):
    """criterion_sparse.py:83-112's sums over the known rows per matched pair (qi, tj int32 [P]) → fp32 [P, 4]:
    Σ focal, Σ σ·t, Σ σ, Σ t.  Differentiable in F [N, Q]; only the pairs' columns get a gradient."""

    @staticmethod
    def forward(ctx, F, bits, T, flags, qi, tj):
        F = F.detach().contiguous()
        P = qi.shape[0]
        out = torch.empty(P, 4, dtype=torch.float32, device=F.device)
        call("pasco_setloss_pair_sums", ptr(F), F.shape[0], F.shape[1], ptr(bits), T, ptr(flags), ptr(qi), ptr(tj), P,
             ptr(out))
        ctx.save_for_backward(F, bits, flags, qi, tj)
        ctx.T = T
        return out

    @staticmethod
    def backward(ctx, g):
        F, bits, flags, qi, tj = ctx.saved_tensors
        gF = torch.zeros_like(F)
        call("pasco_setloss_pair_backward", ptr(F), F.shape[0], F.shape[1], ptr(bits), ctx.T, ptr(flags), ptr(qi),
             ptr(tj), qi.shape[0], ptr(g.contiguous()), ptr(gF))
        return gF, None, None, None, None, None


class SscLogits(torch.autograd.Function):
    """helper.py:7-37's voxel class logits: out [N, K] = normalised (σ(F[:, keep]) + 1e-8) @ L, L = query_logits[keep,
    :-1] [kq, K].  Differentiable in F (kept columns) and L."""

    @staticmethod
    def forward(ctx, F, L, keep):
        F, L = F.detach().contiguous(), L.detach().contiguous()
        out = torch.empty(F.shape[0], L.shape[1], dtype=torch.float32, device=F.device)
        call("pasco_setloss_ssc_forward", ptr(F), F.shape[0], F.shape[1], ptr(keep), keep.shape[0], ptr(L), L.shape[1],
             ptr(out))
        ctx.save_for_backward(F, L, keep, out)
        return out

    @staticmethod
    def backward(ctx, g):
        F, L, keep, out = ctx.saved_tensors
        gF = torch.zeros_like(F)
        gL = torch.empty_like(L)
        call("pasco_setloss_ssc_backward", ptr(F), F.shape[0], F.shape[1], ptr(keep), keep.shape[0], ptr(L), L.shape[1],
             ptr(out), ptr(g.contiguous()), ptr(gF), ptr(gL))
        return gF, gL, None


class LovaszClasses(torch.autograd.Function):
    """lovasz.py:186-219's per-class term Σ err·lovasz_grad for every class at once → fp32 [C].  logits [P, C];
    labels int32 [P] (−1: row left out, >= C: background of every class).  One batched sort of the [C, P] errors."""

    @staticmethod
    def forward(ctx, logits, labels):
        x = logits.detach().contiguous()
        P, C_ = x.shape
        probs = torch.empty_like(x)
        err = torch.empty(C_, P, dtype=torch.float32, device=x.device)
        call("pasco_lovasz_errors", ptr(x), P, C_, ptr(labels), ptr(probs), ptr(err))
        err_sorted, perm = torch.sort(err, dim=1, descending=True)
        grad = torch.empty_like(err)
        loss = torch.empty(C_, dtype=torch.float32, device=x.device)
        call("pasco_lovasz_grad", ptr(err_sorted), ptr(perm), ptr(labels), P, C_, ptr(grad), ptr(loss))
        ctx.save_for_backward(probs, labels, perm, grad)
        return loss

    @staticmethod
    def backward(ctx, g):
        probs, labels, perm, grad = ctx.saved_tensors
        dx = torch.empty_like(probs)
        call("pasco_lovasz_backward", ptr(probs), ptr(labels), ptr(perm), ptr(grad), ptr(g.contiguous().float()),
             probs.shape[0], probs.shape[1], ptr(dx))
        return dx, None


def lovasz_softmax(logits: torch.Tensor, labels: torch.Tensor, present: torch.Tensor) -> torch.Tensor:
    """lovasz.py:186-219 with classes="present": the mean of LovaszClasses over the classes flagged in `present`
    (bool [C], device; the present, non-ignored classes — at least one)."""
    per = LovaszClasses.apply(logits.float(), labels)
    w = present.to(per.dtype)
    return (per * w).sum() / w.sum()


# ------------------------------------------------------------------------------------------------
# the criterion over a table of levels (pasco_setloss_*_group, pasco_lovasz_*_group): one launch per pass for all
# levels; each level's arithmetic and summation order are those of the one-level calls above
# ------------------------------------------------------------------------------------------------
def on_device(t, dev) -> torch.Tensor:
    """t on `dev` without a blocking copy: host tensors or lists (bounds, class weights, target classes) go through
    pinned memory."""
    t = torch.as_tensor(t)
    return t if t.device == dev else t.pin_memory().to(dev, non_blocking=True)


def pinned_to(vals, dtype, dev) -> torch.Tensor:
    """A small host list on `dev` through pinned memory, without waiting for the device."""
    return torch.tensor(vals, dtype=dtype).pin_memory().to(dev, non_blocking=True)


def _group(name: str, struct, rows, *args):
    if rows:
        call(name, _lib.table(struct, rows), len(rows), *args)


def setloss_keep_group(query_logits: Sequence[torch.Tensor]):
    """helper.py:20-23 for every level: query_logits fp32 [Q, K1] each → (keep int32 [L, max Q], kept int32 [L]), the
    ascending indices of the queries whose arg-max is not the last class and their count, per level."""
    dev = query_logits[0].device
    keep = torch.empty(len(query_logits), max(q.shape[0] for q in query_logits), dtype=torch.int32, device=dev)
    kept = torch.empty(len(query_logits), dtype=torch.int32, device=dev)
    _group("pasco_setloss_keep_group", _lib.SetlossLevel,
           [dict(query_logits=q, Q=q.shape[0], K1=q.shape[1], keep=keep[i], kept=kept[i:i + 1])
            for i, q in enumerate(query_logits)])
    return keep, kept


def match_cost_group(levels: Sequence[dict], cost_mask: float, cost_class: float, cost_dice: float) -> torch.Tensor:
    """match_cost for every level: dicts of F, bits, T, flags, stats, query_logits, ids, class_weight (match_cost's
    arguments) → one fp32 buffer holding each level's C [Q, T] in turn."""
    sizes = [lv["F"].shape[1] * lv["T"] for lv in levels]
    out = torch.empty(sum(sizes), dtype=torch.float32, device=levels[0]["F"].device)
    rows, at = [], 0
    for lv, sz in zip(levels, sizes):
        F, ql = lv["F"], lv["query_logits"]
        rows.append(dict(F=F, n=F.shape[0], Q=F.shape[1], T=lv["T"], bits=lv["bits"], flags=lv["flags"],
                         stats=lv["stats"], query_logits=ql, K1=ql.shape[1], ids=lv["ids"],
                         class_weight=lv["class_weight"], C=out[at:at + sz] if sz else None))
        at += sz
    _group("pasco_setloss_match_cost_group", _lib.SetlossLevel, rows, float(cost_mask), float(cost_class),
           float(cost_dice))
    return out


class PairSumsGroup(torch.autograd.Function):
    """PairSums for every level: apply(meta, *F) with meta one (bits, T, flags, qi, tj) per level and F fp32 [N, Q]
    each → fp32 [ΣP, 4], the levels' pairs in turn."""

    @staticmethod
    def forward(ctx, meta, *Fs):
        Fs = [F.detach().contiguous() for F in Fs]
        P = [m[3].shape[0] for m in meta]
        out = torch.empty(sum(P), 4, dtype=torch.float32, device=Fs[0].device)
        ctx.rows = []
        for F, (bits, T, flags, qi, tj), p in zip(Fs, meta, P):
            ctx.rows.append(dict(F=F, n=F.shape[0], Q=F.shape[1], T=T, bits=bits, flags=flags, qi=qi, tj=tj, P=p))
        fwd, at = [], 0
        for row, p in zip(ctx.rows, P):
            if p:
                fwd.append(dict(row, sums=out[at:at + p]))
            at += p
        _group("pasco_setloss_pair_sums_group", _lib.SetlossLevel, fwd)
        ctx.P, ctx.keep_alive = P, (Fs, meta)
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        gFs, rows, at = [], [], 0
        for row, p in zip(ctx.rows, ctx.P):
            gF = torch.zeros_like(row["F"])
            gFs.append(gF)
            if p:
                rows.append(dict(row, g_sums=g[at:at + p], gF_pairs=gF))
            at += p
        _group("pasco_setloss_pair_backward_group", _lib.SetlossLevel, rows)
        return (None, *gFs)


class SscLogitsGroup(torch.autograd.Function):
    """SscLogits for every level, the class logits read through the kept-query list: apply(meta, *F, *query_logits)
    with meta one (keep int32 [≥ kq], kq) per level, F fp32 [N, Q], query_logits fp32 [Q, K+1] → one fp32 [N, K] per
    level, out = normalised (σ(F[:, keep[:kq]]) + 1e-8) @ query_logits[keep[:kq], :K].  Every kq >= 1."""

    @staticmethod
    def forward(ctx, meta, *tensors):
        L = len(meta)
        Fs = [F.detach().contiguous() for F in tensors[:L]]
        qls = [q.detach().contiguous() for q in tensors[L:]]
        outs, rows = [], []
        for F, ql, (keep, kq) in zip(Fs, qls, meta):
            K = ql.shape[1] - 1
            out = torch.empty(F.shape[0], K, dtype=torch.float32, device=F.device)
            outs.append(out)
            rows.append(dict(F=F, n=F.shape[0], Q=F.shape[1], keep=keep, kq=kq, L=ql, L_rows=keep, ldL=ql.shape[1], K=K,
                             ssc=out))
        _group("pasco_setloss_ssc_forward_group", _lib.SetlossLevel, rows)
        ctx.rows, ctx.meta, ctx.keep_alive = rows, meta, (Fs, qls, outs)
        return tuple(outs)

    @staticmethod
    def backward(ctx, *gs):
        rows, gFs, gLs = [], [], []
        for row, g, (keep, kq) in zip(ctx.rows, gs, ctx.meta):
            gF = torch.zeros_like(row["F"])
            gL = torch.empty(kq, row["K"], dtype=torch.float32, device=gF.device)
            gFs.append(gF)
            gLs.append(gL)
            rows.append(dict(row, g_ssc=g.contiguous(), gF_ssc=gF, gL=gL))
        _group("pasco_setloss_ssc_backward_group", _lib.SetlossLevel, rows)
        gqs = []
        for row, gL, (keep, kq) in zip(ctx.rows, gLs, ctx.meta):
            gq = torch.zeros_like(row["L"])
            gq[keep[:kq].long(), :row["K"]] = gL
            gqs.append(gq)
        return (None, *gFs, *gqs)


def _segmented_descending(err: torch.Tensor, shapes: Sequence[Tuple[int, int]]):
    """Sorts each class row of each term's [C, P] errors (the terms laid out in turn in the flat fp32 `err`) descending,
    in one stable sort of int64 keys (row index << 32 | 0x7FFFFFFF − float bits), built in place: non-negative errors
    order as their bits, the −1 of rows left out after all of them.  → (sorted errors, each position's row within its
    term).  Temporaries: the key, the sorted key and the permutation, int64 each, the key freed before the gather."""
    dev = err.device
    key = err.view(torch.int32).to(torch.int64).neg_().add_(0x7FFFFFFF)
    at, row0 = 0, 0
    for C_, P in shapes:
        key[at:at + C_ * P].view(C_, P).add_((torch.arange(row0, row0 + C_, device=dev) << 32).view(C_, 1))
        at, row0 = at + C_ * P, row0 + C_
    perm = torch.sort(key, stable=True)[1]
    del key
    err_sorted = err[perm]
    at = 0
    for C_, P in shapes:
        perm[at:at + C_ * P].view(C_, P).sub_((at + P * torch.arange(C_, device=dev)).view(C_, 1))
        at += C_ * P
    return err_sorted, perm


class LovaszGroup(torch.autograd.Function):
    """LovaszClasses for every term: apply(labels, *logits) with labels one int32 [P] per term (LovaszClasses' label
    convention) and logits fp32 [P, C] → fp32 [ΣC], each term's per-class Σ err·lovasz_grad in turn.  One errors
    launch, one segmented sort of all terms' [C, P] errors, one grad launch."""

    @staticmethod
    def forward(ctx, labels, *logits):
        xs = [x.detach().contiguous() for x in logits]
        dev = xs[0].device
        sizes = [x.numel() for x in xs]
        err = torch.empty(sum(sizes), dtype=torch.float32, device=dev)
        probs = [torch.empty_like(x) for x in xs]
        rows, at = [], 0
        for x, lab, pr, sz in zip(xs, labels, probs, sizes):
            rows.append(dict(logits=x, P=x.shape[0], C=x.shape[1], labels=lab, probs=pr, err=err[at:at + sz]))
            at += sz
        _group("pasco_lovasz_errors_group", _lib.LovaszTerm, rows)
        err_sorted, perm = _segmented_descending(err, [(x.shape[1], x.shape[0]) for x in xs])
        grad = torch.empty_like(err)
        loss = torch.zeros(sum(x.shape[1] for x in xs), dtype=torch.float32, device=dev)     # a term without rows: 0
        grows, at, c0 = [], 0, 0
        for x, lab, sz in zip(xs, labels, sizes):
            C_ = x.shape[1]
            grows.append(dict(P=x.shape[0], C=C_, labels=lab, err_sorted=err_sorted[at:at + sz], perm=perm[at:at + sz],
                              grad=grad[at:at + sz], loss=loss[c0:c0 + C_]))
            at, c0 = at + sz, c0 + C_
        _group("pasco_lovasz_grad_group", _lib.LovaszTerm, [r for r in grows if r["P"] > 0])
        ctx.grows, ctx.keep_alive = grows, (probs, labels, perm, grad)
        ctx.probs = probs
        return loss

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous().float()
        dxs, rows, c0 = [], [], 0
        for r, pr in zip(ctx.grows, ctx.probs):
            dx = torch.zeros_like(pr)
            dxs.append(dx)
            if r["P"] > 0:
                rows.append(dict(probs=pr, labels=r["labels"], perm=r["perm"], grad=r["grad"], g=g[c0:c0 + r["C"]],
                                 P=r["P"], C=r["C"], dx=dx))
            c0 += r["C"]
        _group("pasco_lovasz_backward_group", _lib.LovaszTerm, rows)
        return (None, *dxs)
