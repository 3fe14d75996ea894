"""``SparseConvTensor`` and the cached-rulebook records of the drop-in surface.

Public names, constructor arguments, assertions and method semantics follow
``spconv/pytorch/core.py:60-331`` so model code written against ``spconv.pytorch`` runs
unchanged; the implementation is this project's own (dataclass records, a single
``_derive`` cloning primitive, linear-index densify).
"""
from __future__ import annotations

from contextlib import contextmanager
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from ..constants import SPCONV_FX_TRACE_MODE
from ..core import ConvAlgo

TensorOrSparse = Union["SparseConvTensor", torch.Tensor]


class _NullRegion:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


_NULL_REGION = _NullRegion()


class CUDAKernelTimer:
    """Named CUDA-event regions, active only when ``enable`` (reference ``spconv/tools.py:23-78``)."""

    def __init__(self, enable: bool = True) -> None:
        self.enable = bool(enable)
        self._scope: List[str] = []
        self._events: Dict[str, List[Tuple[torch.cuda.Event, torch.cuda.Event]]] = {}

    def namespace(self, name: str):
        if not self.enable:
            return _NULL_REGION
        return self._namespace(name)

    @contextmanager
    def _namespace(self, name: str):
        self._scope.append(name)
        try:
            yield self
        finally:
            self._scope.pop()

    def record(self, name: str, stream: int = 0):
        if not self.enable:
            return _NULL_REGION          # no generator / context objects on the hot path
        return self._record(name)

    @contextmanager
    def _record(self, name: str):
        begin, finish = (torch.cuda.Event(enable_timing=True) for _ in range(2))
        begin.record()
        try:
            yield self
        finally:
            finish.record()
            self._events.setdefault(".".join([*self._scope, name]), []).append((begin, finish))

    def snapshot(self) -> Tuple[str, ...]:
        """The current namespace stack (autograd Functions keep it so that the backward regions of
        a layer land under the same prefix as its forward regions)."""
        return tuple(self._scope)

    def scoped(self, scope: Sequence[str]):
        if not self.enable:
            return _NULL_REGION
        return self._scoped(scope)

    @contextmanager
    def _scoped(self, scope: Sequence[str]):
        saved = self._scope
        self._scope = list(scope)
        try:
            yield self
        finally:
            self._scope = saved

    def get_all_pair_time(self) -> Dict[str, float]:
        if not self.enable:
            return {}
        torch.cuda.synchronize()
        return {k: sum(b.elapsed_time(f) for b, f in pairs) for k, pairs in self._events.items()}


class ThrustSortAllocator:
    """Keeps one growing scratch buffer alive across rulebook builds
    (role of the reference's thrust temp cache, ``core.py:42-57``)."""

    def __init__(self, device: torch.device) -> None:
        self.device = device
        self._scratch: Optional[torch.Tensor] = None

    def get(self, nbytes: int) -> torch.Tensor:
        if self._scratch is None or self._scratch.numel() < nbytes:
            self._scratch = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=self.device)
        return self._scratch


@dataclass
class IndiceData:
    """Cached ConvAlgo.Native rulebook (fields as ``core.py:60-78``)."""
    out_indices: torch.Tensor
    indices: torch.Tensor
    indice_pairs: torch.Tensor
    indice_pair_num: torch.Tensor
    spatial_shape: List[int]
    out_spatial_shape: List[int]
    is_subm: bool
    algo: ConvAlgo
    ksize: List[int]
    stride: List[int]
    dilation: List[int]
    padding: List[int]
    voxel_num: Optional[Any] = None


@dataclass
class ImplicitGemmIndiceData:
    """Cached masked-implicit-GEMM rulebook (fields as ``core.py:81-112``)."""
    out_indices: torch.Tensor
    indices: torch.Tensor
    pair_fwd: torch.Tensor
    pair_bwd: torch.Tensor
    pair_mask_fwd_splits: List[torch.Tensor]
    pair_mask_bwd_splits: List[torch.Tensor]
    mask_argsort_fwd_splits: List[torch.Tensor]
    mask_argsort_bwd_splits: List[torch.Tensor]
    masks: List[np.ndarray]
    spatial_shape: List[int] = field(default_factory=list)
    out_spatial_shape: List[int] = field(default_factory=list)
    is_subm: bool = False
    algo: ConvAlgo = ConvAlgo.MaskImplicitGemm
    ksize: List[int] = field(default_factory=list)
    stride: List[int] = field(default_factory=list)
    dilation: List[int] = field(default_factory=list)
    padding: List[int] = field(default_factory=list)
    in_voxel_num: Optional[Any] = None
    out_voxel_num: Optional[Any] = None
    # built ahead of the forward pass by RulebookPrefetcher: the only case in which a strided conv may
    # pick its rulebook up from the indice_dict (the reference lets SubM layers alone reuse a key)
    prefetched: bool = False
    # the rulebook of a conv onto given coordinates (SparseConvolution's ``target``): stride / padding are those of
    # the relation (SubM: 1 and (k // 2) * d), ``transposed`` its kind
    cross: bool = False
    transposed: bool = False

    @classmethod
    def from_rulebook(cls, res, indices: torch.Tensor, in_voxel_num, is_subm: bool, **geometry):
        """The entry of the 9-tuple ``res`` of ``ops.get_indice_pairs_implicit_gemm`` built on ``indices``."""
        outids, _, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks = res
        return cls(outids, indices, pair_fwd, pair_bwd, mask_fwd, mask_bwd, sort_fwd, sort_bwd, masks, is_subm=is_subm,
                   in_voxel_num=in_voxel_num, out_voxel_num=_out_voxel_num(outids, in_voxel_num, is_subm), **geometry)


def _out_voxel_num(outids: torch.Tensor, in_voxel_num, is_subm: bool):
    # SubM keeps its input's rows; a bounded rulebook leaves its output count on the device (None: all rows valid)
    return in_voxel_num if is_subm else getattr(outids, "_spx_num_valid", None)


def rulebook_num_valid(outids: torch.Tensor, inp: "SparseConvTensor", out: "SparseConvTensor", is_subm: bool,
                       layer) -> Optional[torch.Tensor]:
    """``num_valid`` of the output ``out`` of a conv / pool ``layer`` on ``inp`` whose rows are ``outids``.  A
    bounded rulebook's status word joins ``out.bound_status`` under the layer's name."""
    num_valid = _out_voxel_num(outids, inp.num_valid, is_subm)
    if num_valid is not None and not is_subm:
        out.bound_status = {**(inp.bound_status or {}), layer._layer_name(): outids._spx_bound_status}
    return num_valid


def scatter_nd(indices: torch.Tensor, updates: torch.Tensor, shape: Sequence[int]) -> torch.Tensor:
    """Dense tensor of ``shape`` with ``updates`` written at integer coordinates ``indices``
    (last-writer-wins on duplicates, as the reference's ``scatter_nd``)."""
    lead = indices.shape[-1]
    dims = [int(s) for s in shape]
    # row-major linear index with host scalars: no host-to-device copy, so a padded ToDense captures
    rows = indices.reshape(-1, lead).long()
    flat = rows[:, 0]
    for a in range(1, lead):
        flat = flat * dims[a] + rows[:, a]
    cells = int(np.prod(dims[:lead]))
    out = updates.new_zeros((cells, *dims[lead:]))
    out[flat] = updates.reshape(-1, *dims[lead:])
    return out.reshape(dims)


class SparseConvTensor:
    """Features ``[N, C]`` + integer coordinates ``[N, ndim+1]`` (batch index first)."""

    # attributes copied verbatim whenever a tensor is re-wrapped
    _CARRIED = ("benchmark", "benchmark_record", "thrust_allocator", "_timer", "force_algo",
                "int8_scale", "fp8_scale")

    def __init__(self, features: torch.Tensor, indices: torch.Tensor,
                 spatial_shape: Union[List[int], np.ndarray], batch_size: int,
                 grid: Optional[torch.Tensor] = None, voxel_num: Optional[torch.Tensor] = None,
                 indice_dict: Optional[dict] = None, benchmark: bool = False,
                 permanent_thrust_allocator: bool = False, enable_timer: bool = False,
                 force_algo: Optional[ConvAlgo] = None):
        if not SPCONV_FX_TRACE_MODE:
            assert features.ndim == 2
            assert indices.ndim == 2
            assert len(spatial_shape) == indices.shape[1] - 1, "spatial shape must equal to ndim"
            assert indices.dtype == torch.int32, "only support int32"
            assert batch_size > 0
        self._features = features
        self.indices = indices
        self.spatial_shape = [int(s) for s in spatial_shape]
        self.batch_size = batch_size
        self.indice_dict = {} if indice_dict is None else indice_dict
        self.grid = torch.Tensor() if grid is None else grid
        self.voxel_num = voxel_num
        self.benchmark = benchmark
        self.benchmark_record: Dict[str, Any] = {}
        self.thrust_allocator = (ThrustSortAllocator(features.device)
                                 if permanent_thrust_allocator else None)
        self._timer = CUDAKernelTimer(enable_timer)
        self.force_algo = force_algo
        self.int8_scale: Optional[np.ndarray] = None
        # float8_e4m3fn features: the per-tensor device scale (fp32 [1]), real value = e4m3 * fp8_scale
        self.fp8_scale: Optional[torch.Tensor] = None
        # padded tensors (bounded rulebooks, pad_to): device int32 [1] = number of valid rows, rows beyond it
        # are padding (indices -1); None = every row is valid.  bound_status: {layer name: status word} of the
        # bounded layers the tensor went through (spconv.check_bounds)
        self.num_valid: Optional[torch.Tensor] = None
        self.bound_status: Optional[Dict[str, torch.Tensor]] = None

    # ------------------------------------------------------------------ cloning
    def _derive(self, features: torch.Tensor) -> "SparseConvTensor":
        """Second handle on the same members with other features.  (Built without re-running the
        constructor's argument checks: this runs twice per layer on the eager path.)"""
        twin = object.__new__(SparseConvTensor)
        twin.__dict__.update(self.__dict__)
        twin._features = features
        return twin

    def replace_feature(self, feature: torch.Tensor) -> "SparseConvTensor":
        """The only way to change features: ``x = x.replace_feature(F.relu(x.features))``."""
        return self._derive(feature)

    def shadow_copy(self) -> "SparseConvTensor":
        """A second handle on the same members (indice_dict shared, not copied)."""
        return self._derive(self._features)

    def select_by_index(self, valid_indices: torch.Tensor) -> "SparseConvTensor":
        picked = self._derive(self._features[valid_indices])
        picked.indices = self.indices[valid_indices]
        picked.indice_dict = {}          # cached rulebooks describe the old coordinate set
        picked.num_valid = None          # the caller picked the rows: padding among them stays inert (indices -1)
        return picked

    # ------------------------------------------------------------------ padding
    def valid_mask(self) -> torch.Tensor:
        """Device bool ``[rows]``: True for valid rows, False for padding (no host sync)."""
        rows = self._features.shape[0]
        dev = self._features.device
        if self.num_valid is None:
            return torch.ones((rows,), dtype=torch.bool, device=dev)
        return torch.arange(rows, dtype=torch.int32, device=dev) < self.num_valid.to(dev)

    def pad_to(self, rows: int) -> "SparseConvTensor":
        """The same tensor with ``rows`` rows: index rows of -1 and zero features are appended and
        ``num_valid`` is set, so inputs of different sizes share one static shape (CUDA-graph replay).
        Sizes are host-known here: no sync.  Cached rulebooks are dropped."""
        n = self._features.shape[0]
        if rows < n:
            raise ValueError(f"pad_to({rows}): the tensor already has {n} rows")
        dev = self._features.device
        feats = torch.cat([self._features, self._features.new_zeros((rows - n, self._features.shape[1]))], 0)
        inds = torch.cat([self.indices, self.indices.new_full((rows - n, self.indices.shape[1]), -1)], 0)
        out = self._derive(feats)
        out.indices = inds
        out.indice_dict = {}
        if self.num_valid is None:
            out.num_valid = torch.full((1,), n, dtype=torch.int32, device=dev)
        return out

    def require_unpadded(self, what: str) -> None:
        if self.num_valid is not None:
            raise NotImplementedError(
                f"padded SparseConvTensor: {what} reduces over rows and is not padding-aware; run it on an "
                "unpadded tensor (no num_out_act_bound / pad_to before it)")

    def minus(self) -> "SparseConvTensor":
        return self._derive(-self._features)

    # ------------------------------------------------------------------ features
    @property
    def features(self) -> torch.Tensor:
        return self._features

    @features.setter
    def features(self, val):
        raise ValueError("you can't set feature directly, use 'x = x.replace_feature("
                         "your_new_feature)' to generate new SparseConvTensor instead.")

    @property
    def is_quantized(self) -> bool:
        return self._features.dtype == torch.qint8

    def q_scale(self):
        if not self.is_quantized:
            raise ValueError("sparse tensor must be quantized")
        return self._features.q_scale()

    def dequantize(self) -> "SparseConvTensor":
        return self._derive(self._features.dequantize())

    # ------------------------------------------------------------------ dense <-> sparse
    @classmethod
    def from_dense(cls, x: torch.Tensor) -> "SparseConvTensor":
        """From a channel-last dense tensor ``(N, *spatial, C)``; zero cells are dropped."""
        coo = x.to_sparse(x.ndim - 1)
        coords = coo.indices().t().contiguous().to(torch.int32)
        return cls(coo.values(), coords, list(coo.shape[1:-1]), int(coo.shape[0]))

    def dense(self, channels_first: bool = True) -> torch.Tensor:
        nd = len(self.spatial_shape)
        full = [self.batch_size, *self.spatial_shape, self._features.shape[1]]
        if self.num_valid is not None:
            # padding rows go to one spare sample that is cut off again: no sync, valid cells untouched
            spare = torch.zeros_like(self.indices[:1])
            spare[:, 0].fill_(self.batch_size)
            inds = torch.where(self.valid_mask().unsqueeze(1), self.indices, spare)
            full[0] += 1
            grid = scatter_nd(inds, self._features, full)[:self.batch_size]
        else:
            grid = scatter_nd(self.indices.to(self._features.device), self._features, full)
        if not channels_first:
            return grid
        return grid.permute(0, nd + 1, *range(1, nd + 1)).contiguous()

    @property
    def spatial_size(self):
        return np.prod(self.spatial_shape)

    def find_indice_pair(self, key) -> Optional[Union[IndiceData, ImplicitGemmIndiceData]]:
        return None if key is None else self.indice_dict.get(key)

    # ------------------------------------------------------------------ arithmetic
    @staticmethod
    def _feat_of(other: TensorOrSparse) -> torch.Tensor:
        assert isinstance(other, (SparseConvTensor, torch.Tensor))
        return other if isinstance(other, torch.Tensor) else other.features

    def __add__(self, other: TensorOrSparse) -> "SparseConvTensor":
        return self._derive(self._features + self._feat_of(other))

    __radd__ = __add__

    def __iadd__(self, other: TensorOrSparse) -> "SparseConvTensor":
        self._features += self._feat_of(other)
        return self

    def __repr__(self) -> str:
        return f"SparseConvTensor[shape={self._features.shape}]"


def expand_nd(ndim: int, val: Union[int, Sequence[int], np.ndarray]) -> List[int]:
    """Scalar or per-axis sequence -> list of ``ndim`` ints."""
    out = [int(val)] * ndim if isinstance(val, (int, np.integer)) else [int(v) for v in val]
    assert len(out) == ndim
    return out
