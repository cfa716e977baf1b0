"""`MinkowskiEngine`-compatible operator surface of the sm_90a engine — the drop-in boundary
(SURVEY.md §8b).  `compat/MinkowskiEngine` re-exports this module so that PaSCo's
`import MinkowskiEngine as ME` resolves here.

Only the live surface of the reference is implemented (call sites cited per symbol); all
sparse work runs in libpasco_sm100.so through pasco_b200.ops — CUDA tensors only, no CPU path.
Module / parameter names follow MinkowskiEngine (`kernel`, `bias`, `.bn.weight`, …) so
reference state_dicts load unchanged.
"""
from __future__ import annotations

import itertools
import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from .. import ops
from ..ops import KernelMap, scatter_max, set_precision, get_precision  # noqa: F401

__version__ = "0.5.4+pasco_b200"


def _triple(v) -> Tuple[int, int, int]:
    if isinstance(v, torch.Tensor):
        v = v.flatten().tolist()
    if isinstance(v, (list, tuple)):
        if len(v) == 1:
            v = list(v) * 3
        assert len(v) == 3
        return tuple(int(x) for x in v)
    return (int(v),) * 3


class CoordinateMapKey:
    """Identity of one coordinate set inside a manager (ME CoordinateMapKey)."""
    _ids = itertools.count()

    def __init__(self, tensor_stride, name: str = ""):
        self.tensor_stride = _triple(tensor_stride)
        self.name = name
        self.uid = next(CoordinateMapKey._ids)

    def get_tensor_stride(self):
        return list(self.tensor_stride)

    def get_key(self):
        return (list(self.tensor_stride), self.name)

    def get_coordinate_size(self):
        return 4

    def __hash__(self):
        return self.uid

    def __eq__(self, other):
        return isinstance(other, CoordinateMapKey) and other.uid == self.uid

    def __repr__(self):
        return f"coordinate map key:{list(self.tensor_stride)}:{self.name or self.uid}"


class _CoordMap:
    __slots__ = ("coords", "table")

    def __init__(self, coords: torch.Tensor, table: Optional[ops.HashTable] = None):
        self.coords = coords
        self.table = table


class CoordinateManager:
    """Owns the coordinate sets (int32 [N,4] in HBM), their hash tables (built lazily) and the
    kernel-map cache shared by every tensor derived from it (unet3d_sparse_v2.py:211,
    decoder_v3.py:145 rely on that sharing)."""

    def __init__(self, D: int = 3, **_):
        self.D = D
        self._maps: Dict[CoordinateMapKey, _CoordMap] = {}
        self._stride_cache: Dict[tuple, tuple] = {}
        self._kmaps: Dict[tuple, KernelMap] = {}

    # -- storage ---------------------------------------------------------------------------------
    def _register(self, coords: torch.Tensor, tensor_stride, table=None) -> CoordinateMapKey:
        key = CoordinateMapKey(tensor_stride)
        self._maps[key] = _CoordMap(coords, table)
        return key

    def get_coordinates(self, key: CoordinateMapKey) -> torch.Tensor:
        return self._maps[key].coords

    def size(self, key: CoordinateMapKey) -> int:
        return self._maps[key].coords.shape[0]

    def _table(self, key: CoordinateMapKey) -> ops.HashTable:
        m = self._maps[key]
        if m.table is None:                       # coordinates of a registered map are unique
            m.table, _ = ops.hash_insert(m.coords)
        return m.table

    def number_of_unique_batch_indices(self) -> int:
        return int(torch.unique(torch.cat([m.coords[:, 0] for m in self._maps.values()])).numel())

    # -- map construction ------------------------------------------------------------------------------
    def insert_and_map(self, coords: torch.Tensor, tensor_stride=1):
        """Dedup (first row wins, order kept).  Returns key, unique_index (None when already unique)."""
        assert coords.is_cuda, "pasco_b200.me: coordinates must be CUDA tensors (no CPU path)"
        coords = coords.to(torch.int32).contiguous()
        n = coords.shape[0]
        table, first = ops.hash_insert(coords)
        keep = first == torch.arange(n, dtype=torch.int32, device=coords.device)
        if bool(keep.all()):
            return self._register(coords, tensor_stride, table), None
        kept, new_row, _ = ops.compact(keep)
        ops.hash_remap(table, new_row)
        return self._register(ops.gather_coords(coords, kept), tensor_stride, table), kept

    def stride(self, in_key: CoordinateMapKey, stride) -> CoordinateMapKey:
        """Coarser map: unique floor(c / s)·s (ME stride map; floors toward −inf)."""
        s = _triple(stride)
        ck = (in_key, s)
        if ck not in self._stride_cache:
            new_ts = tuple(a * b for a, b in zip(in_key.tensor_stride, s))
            child = self._maps[in_key].coords
            floored = ops.coords_floor(child, new_ts)
            table, first = ops.hash_insert(floored)
            keep = first == torch.arange(child.shape[0], dtype=torch.int32, device=child.device)
            kept, new_row, _ = ops.compact(keep)
            ops.hash_remap(table, new_row)
            out_key = self._register(ops.gather_coords(floored, kept), new_ts, table)
            self._stride_cache[ck] = (out_key,)
        return self._stride_cache[ck][0]

    def generate(self, in_key: CoordinateMapKey, kernel_size: int, stride) -> CoordinateMapKey:
        """Generative transposed-conv output map: child row 8·p + k (mink.py:524-527)."""
        assert kernel_size == 2 and _triple(stride) == (2, 2, 2), "only k=2, s=2 is on PaSCo's path"
        ck = (in_key, "gen", kernel_size)
        if ck not in self._stride_cache:
            out_ts = tuple(a // 2 for a in in_key.tensor_stride)
            assert all(a % 2 == 0 for a in in_key.tensor_stride)
            coords = ops.coords_generate_k2(self._maps[in_key].coords, out_ts)
            self._stride_cache[ck] = (self._register(coords, out_ts),)
        return self._stride_cache[ck][0]

    def prune(self, key: CoordinateMapKey, mask: torch.Tensor):
        kept, new_row, total = ops.compact(mask)
        coords = ops.gather_coords(self._maps[key].coords, kept)
        return self._register(coords, key.tensor_stride), kept

    def union_map(self, key_a: CoordinateMapKey, key_b: CoordinateMapKey):
        """Out rows = [A rows ; B rows absent from A].  Returns out_key, rows_b (target row of every B row)."""
        ca, cb = self._maps[key_a].coords, self._maps[key_b].coords
        na = ca.shape[0]
        in_a = ops.hash_lookup(self._table(key_a), cb)
        new = in_a < 0
        kept, new_row, n_new = ops.compact(new)
        rows_b = torch.where(new, new_row + na, in_a).contiguous()
        coords = torch.cat([ca, ops.gather_coords(cb, kept)], 0) if n_new else ca
        return self._register(coords.contiguous(), key_a.tensor_stride), rows_b, na + n_new

    # -- kernel maps ---------------------------------------------------------------------------------------
    def kernel_map(self, in_key, out_key, kernel_size: int, stride: int, dilation: int, transpose: bool) -> KernelMap:
        ck = (in_key, out_key, kernel_size, stride, dilation, transpose)
        km = self._kmaps.get(ck)
        if km is not None:
            return km
        cin, cout = self._maps[in_key].coords, self._maps[out_key].coords
        n_in, n_out = cin.shape[0], cout.shape[0]
        dev = cin.device
        K = kernel_size ** 3
        if transpose:
            # generative k=2,s=2: out row 8p+k ← in row p through W[k]
            assert kernel_size == 2 and stride == 2 and n_out == 8 * n_in
            ar = torch.arange(n_in, dtype=torch.int32, device=dev)
            nbr = torch.full((8, n_in, 8), -1, dtype=torch.int32, device=dev)
            idx = torch.arange(8, device=dev)
            nbr[idx, :, idx] = ar
            nbr = nbr.view(8, n_out)
            nbr_t = torch.arange(n_out, dtype=torch.int32, device=dev).view(n_in, 8).t().contiguous()
            km = KernelMap(nbr, n_in, n_out, nbr_t, list(range(8)))
        elif kernel_size % 2 == 1:
            step = tuple(t * dilation for t in in_key.tensor_stride)
            assert stride == 1, "odd kernels with stride > 1 are not on PaSCo's path"
            nbr = ops.kernel_map_probe(cout, self._table(in_key), kernel_size, step)
            if in_key == out_key:
                km = KernelMap(nbr, n_in, n_out, nbr, [K - 1 - k for k in range(K)])
            else:
                def build_t(self=self, in_key=in_key, out_key=out_key, step=step):
                    t = ops.kernel_map_probe(self._maps[in_key].coords, self._table(out_key), kernel_size, step)
                    return t, [K - 1 - k for k in range(K)]
                km = KernelMap(nbr, n_in, n_out, build_t=build_t)
        else:
            assert kernel_size == stride and dilation == 1, "even kernels: only kernel_size == stride"
            parent_of, slot_of, nbr = ops.kernel_map_down(cin, self._table(out_key), n_out, kernel_size,
                                                          in_key.tensor_stride, want_nbr=True)

            def build_t(parent_of=parent_of, slot_of=slot_of):
                ks = torch.arange(K, dtype=torch.int32, device=dev).view(K, 1)
                t = torch.where(slot_of.view(1, -1) == ks, parent_of.view(1, -1), torch.full_like(parent_of.view(1, -1), -1))
                return t.contiguous(), list(range(K))
            km = KernelMap(nbr, n_in, n_out, build_t=build_t)
            km.parent_of = parent_of
        self._kmaps[ck] = km
        return km

    def pool_map(self, in_key, out_key, kernel_size: int):
        ck = (in_key, out_key, "pool", kernel_size)
        if ck not in self._kmaps:
            parent_of, _, _ = ops.kernel_map_down(self._maps[in_key].coords, self._table(out_key),
                                                  self.size(out_key), kernel_size, in_key.tensor_stride, want_nbr=False)
            self._kmaps[ck] = parent_of
        return self._kmaps[ck]


# ------------------------------------------------------------------------------------------------
# SparseTensor
# ------------------------------------------------------------------------------------------------
class SparseTensorQuantizationMode:
    RANDOM_SUBSAMPLE = 0
    UNWEIGHTED_AVERAGE = 1
    UNWEIGHTED_SUM = 2
    NO_QUANTIZATION = 3
    MAX_POOL = 4


class MinkowskiAlgorithm:
    DEFAULT = 0
    MEMORY_EFFICIENT = 1
    SPEED_OPTIMIZED = 2


class TensorField:
    """Referenced only in isinstance checks (pasco/models/dropout.py:23,47)."""


_HOOKS_PENDING = os.environ.get("PASCO_B200_HOOKS", "0") not in ("", "0")


def _maybe_install_hooks() -> None:
    """PASCO_B200_HOOKS: install the requested hook groups (pasco_b200/hooks.py) once their trigger modules have been
    imported.  Checked when a SparseTensor is built."""
    global _HOOKS_PENDING
    _HOOKS_PENDING = not _hooks._install_requested()


class _LazyRows:
    """Deferred act(BatchNorm(x)) over rows — what MinkowskiBatchNorm (+ a following MinkowskiReLU / LeakyReLU) returns for
    fp32 CUDA rows.  If the consumer is a stride-1 k>1 MinkowskiConvolution the three run through ops.bn_act_conv: in
    training ONE fused node whose BatchNorm apply pass writes the bf16 planes the convolution gathers (ops.BNActConv), in
    eval mode without gradients one split pass with the running statistics; any other consumer reading `.F` materialises
    it through the fused row kernels (ops.batchnorm_rows), activation included.  Results are identical either way; this
    only removes one full read+write of the activations per BatchNorm → convolution pair (pre-activation residual blocks,
    pasco/maskpls/mink.py:618-658), in the unmodified reference model and in net3d.PascoNet alike."""
    ndim = 2

    def __init__(self, bn, x: torch.Tensor, act: int, group):
        self.bn, self.x, self.act, self.group = bn, x, act, group
        self.shape, self.device, self.dtype, self.is_cuda = x.shape, x.device, x.dtype, x.is_cuda
        self.requires_grad = x.requires_grad or (bn.weight is not None and bn.weight.requires_grad)

    def size(self, *a):
        return self.x.size(*a)

    def with_act(self, act: int) -> "_LazyRows":
        return _LazyRows(self.bn, self.x, act, self.group)

    def materialise(self) -> torch.Tensor:
        return ops.batchnorm_rows(self.bn, self.x, self.act, self.group)


class SparseTensor:
    """ME.SparseTensor(features, coordinates=None, tensor_stride=1, coordinate_map_key=None,
    coordinate_manager=None) — call sites: net_panoptic_sparse.py:323; unet3d_sparse_v2.py:207-212;
    decoder_v3.py:141-146; transformer_predictor_v2.py:203-205,231,258-262."""

    def __init__(self, features, coordinates=None, tensor_stride=1, coordinate_map_key=None,
                 coordinate_manager=None, quantization_mode=SparseTensorQuantizationMode.RANDOM_SUBSAMPLE,
                 allocator_type=None, minkowski_algorithm=None, requires_grad=None, device=None):
        if not (isinstance(features, (torch.Tensor, _LazyRows)) and features.ndim == 2):
            raise ValueError("features must be a [N, C] tensor")
        if _HOOKS_PENDING:
            _maybe_install_hooks()
        if coordinate_map_key is None:
            if coordinates is None:
                raise ValueError("either coordinates or coordinate_map_key is required")
            if coordinates.ndim != 2 or coordinates.shape[1] != 4 or coordinates.dtype.is_floating_point:
                raise ValueError("coordinates must be an integer [N, 4] tensor (batch, x, y, z)")
            if coordinates.shape[0] != features.shape[0]:
                raise ValueError("coordinates and features disagree on the number of rows")
            if coordinate_manager is None:
                coordinate_manager = CoordinateManager()
            coordinates = coordinates.to(features.device)
            coordinate_map_key, uidx = coordinate_manager.insert_and_map(coordinates, tensor_stride)
            if uidx is not None:
                features = ops.GatherRows.apply(features, uidx)
        else:
            if coordinate_manager is None:
                raise ValueError("coordinate_map_key needs its coordinate_manager")
            if coordinate_manager.size(coordinate_map_key) != features.shape[0]:
                raise RuntimeError("features do not match the size of the coordinate map")
        self._F = features
        self.coordinate_manager = coordinate_manager
        self.coordinate_map_key = coordinate_map_key
        if requires_grad is not None:
            self.F.requires_grad_(requires_grad)

    @property
    def F(self) -> torch.Tensor:
        if isinstance(self._F, _LazyRows):
            self._F = self._F.materialise()
        return self._F

    features = F
    C = property(lambda self: self.coordinate_manager.get_coordinates(self.coordinate_map_key))
    coordinates = C
    tensor_stride = property(lambda self: list(self.coordinate_map_key.tensor_stride))
    D = dimension = property(lambda self: 3)
    shape = property(lambda self: self._F.shape)
    device = property(lambda self: self._F.device)
    dtype = property(lambda self: self._F.dtype)
    requires_grad = property(lambda self: self._F.requires_grad)

    def size(self, *a):
        return self._F.size(*a)

    def __len__(self):
        return self._F.shape[0]

    def __repr__(self):
        return f"SparseTensor(pasco_b200, F={tuple(self._F.shape)}, tensor_stride={self.tensor_stride})"

    def _pending(self) -> Optional[_LazyRows]:
        return self._F if isinstance(self._F, _LazyRows) else None

    # criterion_sparse.py:273-274
    def _rows_of_batch(self, b: int):
        return torch.nonzero(self.C[:, 0] == b, as_tuple=True)[0]

    def features_at(self, b: int):
        return self.F[self._rows_of_batch(b)]

    def coordinates_at(self, b: int):
        return self.C[self._rows_of_batch(b)][:, 1:]

    @property
    def decomposed_features(self):
        nb = int(self.C[:, 0].max()) + 1 if len(self) else 0
        return [self.features_at(b) for b in range(nb)]

    @property
    def decomposed_coordinates(self):
        nb = int(self.C[:, 0].max()) + 1 if len(self) else 0
        return [self.coordinates_at(b) for b in range(nb)]

    def dense(self, shape=None, min_coordinate=None, contract_stride=True):
        """→ (dense [B,C,X,Y,Z], min_coordinate, tensor_stride)  (augmenter.py:15-17;
        unet3d_sparse_v2.py:196-198; transformer_predictor_v2.py:263-274; net_panoptic_sparse.py:453)."""
        C_ = self.C
        ts = self.tensor_stride
        if min_coordinate is None:
            mn = C_[:, 1:].min(0)[0]
            if bool((mn < 0).any()):
                raise ValueError(f"Coordinate has a negative value: {mn}. Please provide min_coordinate argument")
            ret_min = mn.view(1, -1)
            mn_l = [0, 0, 0]
        elif isinstance(min_coordinate, int) and min_coordinate == 0:
            ret_min, mn_l = 0, [0, 0, 0]
        else:
            if not (isinstance(min_coordinate, torch.Tensor) and not min_coordinate.dtype.is_floating_point):
                raise ValueError("min_coordinate must be an IntTensor")
            mn_l = [int(v) for v in min_coordinate.flatten().tolist()]
            ret_min = min_coordinate.view(1, -1) if min_coordinate.ndim == 1 else min_coordinate
        if any(m % s for m, s in zip(mn_l, ts)):
            raise AssertionError("The minimum coordinates must be divisible by the tensor stride.")
        step = ts if contract_stride else [1, 1, 1]
        nch = self.F.shape[1]
        if shape is None:
            mx = C_[:, 1:].max(0)[0].tolist()
            size = [(int(m) - lo) // st + 1 for m, lo, st in zip(mx, mn_l, step)]
            shape = (int(C_[:, 0].max()) + 1, nch, *size)
        else:
            if len(shape) != 5 or int(shape[1]) != nch:
                raise ValueError("shape must be [B, C, X, Y, Z] with C matching the features")
            shape = tuple(int(s) for s in shape)
        dense = ops.ToDense.apply(self.F.float(), C_, tuple(mn_l), tuple(step), shape)
        return dense, ret_min, torch.IntTensor(ts)

    # -- arithmetic: same key → elementwise, different keys → coordinate union (decoder_v3.py:163) --
    def _combine(self, other, sign: float):
        cm = self.coordinate_manager
        if not isinstance(other, SparseTensor):
            return SparseTensor(self.F + sign * other, coordinate_map_key=self.coordinate_map_key, coordinate_manager=cm)
        if other.coordinate_manager is not cm:
            raise ValueError("SparseTensors of different coordinate managers cannot be combined")
        if other.coordinate_map_key == self.coordinate_map_key:
            return SparseTensor(self.F + sign * other.F, coordinate_map_key=self.coordinate_map_key,
                                coordinate_manager=cm)
        out_key, rows_b, n_out = cm.union_map(self.coordinate_map_key, other.coordinate_map_key)
        b = other.F if sign > 0 else -other.F
        return SparseTensor(ops.UnionAdd.apply(self.F.float(), b.float(), rows_b, n_out),
                            coordinate_map_key=out_key, coordinate_manager=cm)

    def __add__(self, other):
        return self._combine(other, 1.0)

    __iadd__ = __add__

    def __sub__(self, other):
        return self._combine(other, -1.0)

    def __mul__(self, other):
        if isinstance(other, SparseTensor):
            assert other.coordinate_map_key == self.coordinate_map_key
            other = other.F
        return SparseTensor(self.F * other, coordinate_map_key=self.coordinate_map_key,
                            coordinate_manager=self.coordinate_manager)

    def detach(self):
        return SparseTensor(self.F.detach(), coordinate_map_key=self.coordinate_map_key,
                            coordinate_manager=self.coordinate_manager)


def _like(x: SparseTensor, feats: torch.Tensor) -> SparseTensor:
    return SparseTensor(feats, coordinate_map_key=x.coordinate_map_key, coordinate_manager=x.coordinate_manager)


# ------------------------------------------------------------------------------------------------
# modules
# ------------------------------------------------------------------------------------------------
class MinkowskiModuleBase(nn.Module):
    pass


class _Convolution(MinkowskiModuleBase):
    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, bias=False,
                 kernel_generator=None, is_transpose=False, expand_coordinates=False, convolution_mode=None,
                 dimension=None):
        super().__init__()
        if dimension not in (None, 3):
            raise ValueError("pasco_b200.me supports dimension=3 only")
        self.in_channels, self.out_channels = int(in_channels), int(out_channels)
        self.kernel_size, self.stride, self.dilation = int(kernel_size), int(stride), int(dilation)
        self.is_transpose, self.expand_coordinates = is_transpose, expand_coordinates
        self.kernel_volume = self.kernel_size ** 3
        self.use_mm = self.kernel_volume == 1 and self.stride == 1
        shape = (self.in_channels, self.out_channels) if self.use_mm else \
            (self.kernel_volume, self.in_channels, self.out_channels)
        self.kernel = nn.Parameter(torch.empty(*shape))
        self.bias = nn.Parameter(torch.empty(1, self.out_channels)) if bias else None
        self._packs = ops.PackedWeights()
        self.reset_parameters()

    def reset_parameters(self):
        fan = (self.out_channels if self.is_transpose else self.in_channels) * self.kernel_volume
        bound = 1.0 / math.sqrt(fan)
        with torch.no_grad():
            self.kernel.uniform_(-bound, bound)
            if self.bias is not None:
                self.bias.uniform_(-bound, bound)

    def forward(self, x: SparseTensor) -> SparseTensor:
        if x.shape[1] != self.in_channels:
            raise RuntimeError(f"Channel size mismatch {x.shape[1]} != {self.in_channels}")
        cm, in_key = x.coordinate_manager, x.coordinate_map_key
        if self.use_mm:
            # ME does F.mm here; tall inputs with 64-multiple channels take the wgmma GEMM (ops.LinearTC), the rest
            # stays the fp32 library GEMM
            out = ops.linear(x.F, self.kernel.t(), self.bias.view(-1) if self.bias is not None else None)
            return SparseTensor(out, coordinate_map_key=in_key, coordinate_manager=cm)
        if self.is_transpose:
            if not self.expand_coordinates:
                raise NotImplementedError("only generative (expand_coordinates=True) transposed conv is on the path")
            out_key = cm.generate(in_key, self.kernel_size, self.stride)
        elif self.stride > 1:
            out_key = cm.stride(in_key, self.stride)
        else:
            out_key = in_key
        kmap = cm.kernel_map(in_key, out_key, self.kernel_size, self.stride, self.dilation, self.is_transpose)
        lazy = x._pending()
        if lazy is not None and out_key == in_key and not self.is_transpose and lazy.dtype == torch.float32:
            out = ops.bn_act_conv(lazy.bn, lazy.x, lazy.act, lazy.group, self.kernel, self.bias, kmap, self._packs)
        else:
            out = ops.SparseConv.apply(x.F.float(), self.kernel, self.bias, kmap, self._packs)
        return SparseTensor(out, coordinate_map_key=out_key, coordinate_manager=cm)

    def extra_repr(self):
        return (f"in={self.in_channels}, out={self.out_channels}, kernel_size={self.kernel_size}, "
                f"stride={self.stride}, dilation={self.dilation}")


class MinkowskiConvolution(_Convolution):
    """mink.py:509-511 (k=2,s=2), 625-638 (k=3); encoder_v2.py:109-111, decoder_v3.py:103-105,133-135 (k=1)."""

    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, bias=False,
                 kernel_generator=None, expand_coordinates=False, convolution_mode=None, dimension=None):
        super().__init__(in_channels, out_channels, kernel_size, stride, dilation, bias, kernel_generator, False,
                         expand_coordinates, convolution_mode, dimension)


class MinkowskiConvolutionTranspose(_Convolution):
    """mink.py:524-527 (k=2, s=2, expand_coordinates=True)."""

    def __init__(self, in_channels, out_channels, kernel_size=-1, stride=1, dilation=1, bias=False,
                 kernel_generator=None, expand_coordinates=False, convolution_mode=None, dimension=None):
        super().__init__(in_channels, out_channels, kernel_size, stride, dilation, bias, kernel_generator, True,
                         expand_coordinates, convolution_mode, dimension)


class MinkowskiBatchNorm(MinkowskiModuleBase):
    """BatchNorm1d over all rows, kept as `.bn` for state-dict compatibility (mink.py:512,528,623,631)."""

    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True):
        super().__init__()
        self.bn = nn.BatchNorm1d(num_features, eps=eps, momentum=momentum, affine=affine,
                                 track_running_stats=track_running_stats)

    def _group(self):
        return None

    def forward(self, x):
        # training-mode statistics + apply run in the fused row kernels (ops.BatchNormAct; the convolution that produced
        # x already left its column sums); same parameters, buffers and running-statistics update as nn.BatchNorm1d.  The
        # deferred form lets a following activation fold into the apply pass and a following stride-1 convolution take
        # bn_act_conv's fusion in every mode (ops.bn_act_conv_route picks it)
        xf = x.F
        if self.bn.running_mean is not None and xf.is_cuda and xf.dtype == torch.float32:
            return _like(x, _LazyRows(self.bn, xf, ops.ACT_NONE, self._group()))      # see _LazyRows
        return _like(x, ops.batchnorm_rows(self.bn, xf, ops.ACT_NONE, self._group()))


class MinkowskiSyncBatchNorm(MinkowskiBatchNorm):
    def __init__(self, num_features, eps=1e-5, momentum=0.1, affine=True, track_running_stats=True,
                 process_group=None):
        MinkowskiModuleBase.__init__(self)
        self.bn = nn.SyncBatchNorm(num_features, eps=eps, momentum=momentum, affine=affine,
                                   track_running_stats=track_running_stats, process_group=process_group)

    def _group(self):
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()) or not self.bn.training:
            return None
        g = self.bn.process_group if self.bn.process_group is not None else dist.group.WORLD
        return g if dist.get_world_size(g) > 1 else None

    @classmethod
    def convert_sync_batchnorm(cls, module, process_group=None):
        """unet3d_sparse_v2.py:172-175."""
        if isinstance(module, MinkowskiBatchNorm) and not isinstance(module, MinkowskiSyncBatchNorm):
            new = cls(module.bn.num_features, module.bn.eps, module.bn.momentum, module.bn.affine,
                      module.bn.track_running_stats, process_group)
            if module.bn.affine:
                new.bn.weight, new.bn.bias = module.bn.weight, module.bn.bias
            new.bn.running_mean, new.bn.running_var = module.bn.running_mean, module.bn.running_var
            new.bn.num_batches_tracked = module.bn.num_batches_tracked
            return new.train(module.training)
        for name, child in module.named_children():
            module.add_module(name, cls.convert_sync_batchnorm(child, process_group))
        return module


def _pointwise(name: str, torch_cls):
    class _Op(MinkowskiModuleBase):
        def __init__(self, *a, **k):
            super().__init__()
            self.module = torch_cls(*a, **k)

        def forward(self, x):
            return _like(x, self.module(x.F))
    _Op.__name__ = _Op.__qualname__ = name
    return _Op


def _activation(name: str, torch_cls, act_code: int):
    base = _pointwise(name, torch_cls)

    class _Act(base):
        def forward(self, x):
            lazy = x._pending()
            if lazy is not None and lazy.act == ops.ACT_NONE and \
                    (act_code != ops.ACT_LEAKY or abs(self.module.negative_slope - 0.01) < 1e-12):
                return _like(x, lazy.with_act(act_code))          # folded into the pending BatchNorm apply
            return base.forward(self, x)
    _Act.__name__ = _Act.__qualname__ = name
    return _Act


MinkowskiReLU = _activation("MinkowskiReLU", nn.ReLU, ops.ACT_RELU)
MinkowskiLeakyReLU = _activation("MinkowskiLeakyReLU", nn.LeakyReLU, ops.ACT_LEAKY)
MinkowskiSigmoid = _pointwise("MinkowskiSigmoid", nn.Sigmoid)
MinkowskiSoftmax = _pointwise("MinkowskiSoftmax", nn.Softmax)
MinkowskiDropout = _pointwise("MinkowskiDropout", nn.Dropout)
MinkowskiGELU = _pointwise("MinkowskiGELU", nn.GELU)
MinkowskiTanh = _pointwise("MinkowskiTanh", nn.Tanh)


class MinkowskiLinear(MinkowskiModuleBase):
    def __init__(self, in_features, out_features, bias=True):
        super().__init__()
        self.linear = nn.Linear(in_features, out_features, bias=bias)

    def forward(self, x):
        return _like(x, self.linear(x.F))


class MinkowskiPruning(MinkowskiModuleBase):
    """Order-preserving row compaction + new coordinate map (decoder_v3.py:127,159,285,421,496; misc.py:17-26)."""

    def forward(self, x: SparseTensor, mask: torch.Tensor) -> SparseTensor:
        if not isinstance(mask, torch.Tensor) or mask.dtype != torch.bool:
            raise TypeError("MinkowskiPruning: mask must be a bool tensor")
        if mask.ndim != 1 or mask.shape[0] != x.F.shape[0]:
            raise RuntimeError(f"MinkowskiPruning: mask length {tuple(mask.shape)} != number of rows {x.F.shape[0]}")
        cm = x.coordinate_manager
        key, kept = cm.prune(x.coordinate_map_key, mask.to(x.F.device))
        return SparseTensor(ops.GatherRows.apply(x.F.float(), kept), coordinate_map_key=key, coordinate_manager=cm)


class MinkowskiMaxPooling(MinkowskiModuleBase):
    """kernel_size == stride local max over existing children (transformer_predictor_v2.py:100-102)."""

    def __init__(self, kernel_size, stride=1, dilation=1, kernel_generator=None, dimension=None):
        super().__init__()
        self.kernel_size, self.stride = int(kernel_size), int(stride)
        if self.kernel_size != self.stride or dilation != 1:
            raise NotImplementedError("pasco_b200.me: max pooling needs kernel_size == stride, dilation 1")

    def forward(self, x: SparseTensor) -> SparseTensor:
        cm, in_key = x.coordinate_manager, x.coordinate_map_key
        if self.stride == 1:
            return x
        out_key = cm.stride(in_key, self.stride)
        parent_of = cm.pool_map(in_key, out_key, self.kernel_size)
        out = ops.MaxPoolRows.apply(x.F.float(), parent_of, cm.size(out_key))
        return SparseTensor(out, coordinate_map_key=out_key, coordinate_manager=cm)


class _NotOnPath(MinkowskiModuleBase):
    """Symbols that only occur in never-instantiated reference classes (SURVEY.md §8b, last table row)."""

    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError(f"{type(self).__name__} is not on PaSCo's live path and is not implemented")


class MinkowskiGlobalPooling(_NotOnPath):
    pass


class MinkowskiGlobalMaxPooling(_NotOnPath):
    pass


class MinkowskiBroadcastMultiplication(_NotOnPath):
    pass


class MinkowskiChannelwiseConvolution(_NotOnPath):
    pass


class MinkowskiPoolingTranspose(_NotOnPath):
    pass


def cat(*tensors):
    if len(tensors) == 1 and isinstance(tensors[0], (list, tuple)):
        tensors = tensors[0]
    k = tensors[0].coordinate_map_key
    if any(t.coordinate_map_key != k for t in tensors):
        raise ValueError("ME.cat: tensors must share a coordinate map")
    return _like(tensors[0], torch.cat([t.F for t in tensors], 1))


def to_sparse(x: torch.Tensor, format=None, coordinates=None, device=None) -> SparseTensor:
    """dense [B,C,X,Y,Z] → rows where Σ_c|x| ≠ 0 in (b,x,y,z) order (augmenter.py:22;
    unet3d_sparse_v2.py:202; ensembler.py:117)."""
    if x.ndim != 5:
        raise ValueError("to_sparse expects a [B, C, X, Y, Z] tensor")
    x = x.contiguous().float()
    B, _, X, Y, Z = x.shape
    if coordinates is None:
        occ = ops.dense_occupancy(x.detach())
        kept, _, _ = ops.compact(occ)
        lin = kept.long()
        z = lin % Z
        y = (lin // Z) % Y
        xx = (lin // (Z * Y)) % X
        b = lin // (Z * Y * X)
        coordinates = torch.stack([b, xx, y, z], 1).to(torch.int32).contiguous()
    else:
        coordinates = coordinates.to(device=x.device, dtype=torch.int32).contiguous()
    feats = ops.FromDense.apply(x, coordinates, (0, 0, 0), (1, 1, 1))
    return SparseTensor(feats, coordinates=coordinates)


class _Utils:
    @staticmethod
    def batched_coordinates(coords: List[torch.Tensor], dtype=torch.int32, device=None):
        """transformer_predictor_v2.py:230,254-256; criterion_sparse.py:275; ensembler.py:54."""
        rows = []
        for b, c in enumerate(coords):
            c = torch.as_tensor(c)
            rows.append(torch.cat([torch.full((c.shape[0], 1), b, dtype=c.dtype, device=c.device), c], 1))
        out = torch.cat(rows, 0).to(dtype) if rows else torch.zeros(0, 4, dtype=dtype)
        return out if device is None else out.to(device)

    @staticmethod
    def sparse_collate(coords, feats, labels=None, dtype=torch.int32, device=None):
        bc = _Utils.batched_coordinates(coords, dtype, device)
        f = torch.cat([torch.as_tensor(x) for x in feats], 0)
        return (bc, f) if labels is None else (bc, f, torch.cat([torch.as_tensor(x) for x in labels], 0))


utils = _Utils()


# last, as hooks imports this module: importing hooks parses PASCO_B200_HOOKS and raises on an unknown group
if _HOOKS_PENDING:
    from .. import hooks as _hooks  # noqa: E402
