"""Point cloud -> voxel front end (``spconv/pytorch/utils.py:23-176``): ``PointToVoxel`` and
``gather_features_by_pc_voxel_id``, plus ``MaskedPointToVoxel``, ``PointVoxelScatter`` and the way back,
``VoxelPointInterpolator`` with ``grid_positions``.  CUDA only; the kernels live in ``csrc/pointops.cu``,
``csrc/point_scatter.cu`` and ``csrc/point_interp.cu``.

Unlike the reference's GPU generator (atomic appends: voxel order and the points kept per voxel
depend on scheduling) the result is deterministic and equal to the reference's CPU generator
(``Point2VoxelCPU``, ``spconv/csrc/sparse/pointops.py:589-695``): voxels are numbered by their first
point, a voxel keeps its first ``max_num_points_per_voxel`` points, both in input order.  A point is
in a voxel when ``floor((p - lo) / vsize)`` (fp32) is a finite value in ``[0, grid)`` on every axis; a
point with a NaN or infinite coordinate gets ``pc_voxel_id`` -1 and makes no voxel.
"""
from __future__ import annotations

import ctypes
from typing import List, Optional, Union

import numpy as np
import torch

from .. import _cabi
from . import functional as Fsp
from . import ops


def calc_point2voxel_meta_data(vsize_xyz: List[float], coors_range_xyz: List[float]):
    """``Point2VoxelCommon::calc_meta_data`` (``pointops.py:42-88``): xyz inputs -> zyx-ordered
    ``(vsize, grid_size, grid_stride, coors_range)``; grid size = round((hi - lo) / vsize) in fp32."""
    nd = len(vsize_xyz)
    assert len(coors_range_xyz) == 2 * nd
    vsize = np.zeros(nd, np.float32)
    rng = np.zeros(2 * nd, np.float32)
    for i in range(nd):
        vsize[nd - 1 - i] = np.float32(vsize_xyz[i])
        rng[nd - 1 - i] = np.float32(coors_range_xyz[i])
        rng[2 * nd - 1 - i] = np.float32(coors_range_xyz[i + nd])
    grid = [int(np.round((rng[nd + i] - rng[i]) / vsize[i])) for i in range(nd)]       # fp32 arithmetic + std::round
    stride, prod = [0] * nd, 1
    for i in range(nd - 1, -1, -1):
        stride[i] = prod
        prod *= grid[i]
    return [float(v) for v in vsize], grid, stride, [float(v) for v in rng]


class PointToVoxel(object):
    """WARNING: construct AFTER selecting the device (same contract as the reference)."""

    def __init__(self, vsize_xyz: List[float], coors_range_xyz: List[float], num_point_features: int,
                 max_num_voxels: int, max_num_points_per_voxel: int,
                 device: torch.device = torch.device("cuda:0")):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("spconv_b200.PointToVoxel: CUDA only (the CPU generator under oracle/ is test "
                               "infrastructure)")
        self.ndim = len(vsize_xyz)
        self.device = device
        self.vsize, self.grid_size, self.grid_stride, self.coors_range = calc_point2voxel_meta_data(
            vsize_xyz, coors_range_xyz)
        self.num_point_features = num_point_features
        self.max_num_voxels = max_num_voxels
        self.max_num_points_per_voxel = max_num_points_per_voxel
        self.voxels = torch.zeros([max_num_voxels, max_num_points_per_voxel, num_point_features],
                                  dtype=torch.float32, device=device)
        self.indices = torch.zeros([max_num_voxels, self.ndim], dtype=torch.int32, device=device)
        self.num_per_voxel = torch.zeros([max_num_voxels], dtype=torch.int32, device=device)
        self._c_vsize = (ctypes.c_float * self.ndim)(*self.vsize)
        self._c_grid = (ctypes.c_int * self.ndim)(*self.grid_size)
        self._c_range = (ctypes.c_float * (2 * self.ndim))(*self.coors_range)

    def __call__(self, pc: torch.Tensor, clear_voxels: bool = True, empty_mean: bool = False):
        """-> ``(voxels [M, max_points, F], indices [M, ndim] (zyx), num_per_voxel [M])``"""
        res = self.generate_voxel_with_id(pc, clear_voxels, empty_mean)
        return res[0], res[1], res[2]

    def generate_voxel_with_id(self, pc: torch.Tensor, clear_voxels: bool = True, empty_mean: bool = False):
        """-> ``(voxels, indices, num_per_voxel, pc_voxel_id [N] int64, -1 = no voxel)``"""
        assert pc.device.type == self.device.type, "your pc device is wrong"
        assert pc.dim() == 2 and pc.shape[1] == self.num_point_features, \
            "your points num features doesn't equal to voxel."
        lib = _cabi.load()
        pc = pc.contiguous().float()
        n = pc.shape[0]
        stream = torch.cuda.current_stream().cuda_stream
        with torch.no_grad():
            pc_voxel_id = torch.empty([n], dtype=torch.int64, device=self.device)
            ws = torch.empty(lib.spx_point2voxel_workspace_size(n, self.ndim), dtype=torch.uint8, device=self.device)
            m_host, tot_host = ctypes.c_int64(0), ctypes.c_int64(0)
            _cabi.check(lib.spx_point2voxel_stage1(pc.data_ptr() if n else None, n, self.num_point_features, self.ndim, 1,
                                                   self._c_vsize, self._c_grid, self._c_range, self.max_num_voxels,
                                                   ctypes.byref(m_host), ctypes.byref(tot_host), ws.data_ptr(),
                                                   ws.numel(), stream), "point2voxel_stage1")
            num_voxels = int(m_host.value)
            if clear_voxels:
                self.voxels.zero_()
            _cabi.check(lib.spx_point2voxel_stage2(pc.data_ptr() if n else None, n, self.num_point_features, self.ndim, 1,
                                                   self._c_vsize, self._c_grid, self._c_range, num_voxels,
                                                   int(tot_host.value), self.max_num_points_per_voxel,
                                                   int(bool(empty_mean)), self.voxels.data_ptr(),
                                                   self.indices.data_ptr(), self.num_per_voxel.data_ptr(),
                                                   pc_voxel_id.data_ptr() if n else None, ws.data_ptr(), ws.numel(),
                                                   stream), "point2voxel_stage2")
            return (self.voxels[:num_voxels].clone(), self.indices[:num_voxels].clone(),
                    self.num_per_voxel[:num_voxels].clone(), pc_voxel_id)


class MaskedPointToVoxel(object):
    """A batch of clouds -> voxels in one call, at static shapes and with no host read-back, so a step from raw
    points to the loss captures as one CUDA graph (``spconv.graph_capture``).

    ``voxels, indices, num_per_voxel, pc_voxel_id, num_valid = gen(points, point_offsets=None, empty_mean=False)``

    * ``points [P, F]`` fp32 on the device; ``point_offsets`` device int32 ``[batch_size + 1]``: sample b owns the
      rows ``[off[b], off[b+1])``.  The offsets are not checked on the host (that would be a read-back); each is
      clamped to ``[0, P]`` and then the prefix maximum is taken, so samples are disjoint and contiguous and a
      decreasing offset gives an empty sample.  Rows outside every sample (e.g. at or beyond ``off[B]``) are
      padding and are never read.  ``None``: one sample made of all P rows.
    * Per sample, the voxels are those of ``PointToVoxel(..., max_num_voxels, ...)`` run on that sample's rows
      alone, bit for bit: first-touch order, the per-sample cap, the first ``max_num_points_per_voxel`` points
      of a voxel, the ``empty_mean`` fill, no voxel for NaN / infinite / out-of-range points.
    * Outputs (``bound = max_num_voxels_total``, default ``batch_size * max_num_voxels``, which never truncates):
      ``voxels [bound, max_points, F]``, ``indices [bound, 1 + ndim]`` int32 (batch index first, then the cell in
      zyx order: the ``SparseConvTensor`` layout), ``num_per_voxel [bound]`` int32, ``pc_voxel_id [P]`` int64 (the
      output row of the point's voxel, -1 for padding points, points without a voxel and points of dropped
      voxels) and ``num_valid [1]`` int32 on the device.  Rows are sample 0's kept voxels, then sample 1's, ..,
      packed; ``M = num_valid = min(sum_b min(count_b, max_num_voxels), bound)``.  Rows ``[M, bound)`` are padding:
      indices -1, voxels 0, num_per_voxel 0.  Every element is written on every call.
    * ``voxels`` / ``indices`` / ``num_per_voxel`` / ``num_valid`` are buffers allocated once by the constructor
      and overwritten by every call (clone them to keep a result); ``pc_voxel_id`` is new per call.
    * With ``max_num_voxels_total < batch_size * max_num_voxels``, voxels ranked at or beyond the bound are dropped
      (deterministically: the first ``bound`` rows of the untruncated result are kept) and bit 0 of the status
      word ``_bound_status`` is set; ``spconv.check_bounds(gen)`` reads it, clears it, and raises.

    The padded ``SparseConvTensor`` of the conv path is the rows with ``num_valid`` attached, e.g. with SECOND's
    mean features (MeanVFE; plain torch, padding rows give 0)::

        voxels, indices, num_per_voxel, pc_voxel_id, num_valid = gen(points, offsets)
        feats = voxels.sum(1) / num_per_voxel.clamp(min=1)[:, None].to(voxels.dtype)
        x = spconv.SparseConvTensor(feats, indices, gen.grid_size, gen.batch_size)
        x.num_valid = num_valid

    A dynamic VFE, which reduces every point of a voxel rather than the first ``max_num_points_per_voxel``, uses
    ``pc_voxel_id`` with :class:`PointVoxelScatter` instead (see its docstring).

    At most ``SPX_P2V_MAX_BATCH`` (65536) samples; P and the bound below 2^31 - 1.  CUDA only.
    """

    def __init__(self, vsize_xyz: List[float], coors_range_xyz: List[float], num_point_features: int,
                 max_num_voxels: int, max_num_points_per_voxel: int, batch_size: int,
                 max_num_voxels_total: Optional[int] = None, device: torch.device = torch.device("cuda:0")):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("spconv_b200.MaskedPointToVoxel: CUDA only")
        if max_num_voxels <= 0 or max_num_points_per_voxel <= 0 or batch_size <= 0:
            raise ValueError("MaskedPointToVoxel: max_num_voxels, max_num_points_per_voxel and batch_size must be "
                             "positive")
        if batch_size > _cabi.SPX_P2V_MAX_BATCH:
            raise ValueError(f"MaskedPointToVoxel: batch_size {batch_size} above {_cabi.SPX_P2V_MAX_BATCH}")
        bound = batch_size * max_num_voxels if max_num_voxels_total is None else int(max_num_voxels_total)
        if bound <= 0 or bound >= 2 ** 31 - 1:
            raise ValueError(f"MaskedPointToVoxel: max_num_voxels_total {bound} not in [1, 2^31 - 2]")
        self.ndim = len(vsize_xyz)
        self.device = device
        self.vsize, self.grid_size, self.grid_stride, self.coors_range = calc_point2voxel_meta_data(
            vsize_xyz, coors_range_xyz)
        self.num_point_features = num_point_features
        self.max_num_voxels = max_num_voxels
        self.max_num_points_per_voxel = max_num_points_per_voxel
        self.batch_size = batch_size
        self.max_num_voxels_total = bound
        self.voxels = torch.zeros([bound, max_num_points_per_voxel, num_point_features], dtype=torch.float32,
                                  device=device)
        self.indices = torch.full([bound, 1 + self.ndim], -1, dtype=torch.int32, device=device)
        self.num_per_voxel = torch.zeros([bound], dtype=torch.int32, device=device)
        self.num_valid = torch.zeros([1], dtype=torch.int32, device=device)
        self._bound_status = torch.zeros([1], dtype=torch.int32, device=device)
        self._c_vsize = (ctypes.c_float * self.ndim)(*self.vsize)
        self._c_grid = (ctypes.c_int * self.ndim)(*self.grid_size)
        self._c_range = (ctypes.c_float * (2 * self.ndim))(*self.coors_range)

    def __call__(self, points: torch.Tensor, point_offsets: Optional[torch.Tensor] = None, empty_mean: bool = False):
        if not points.is_cuda or (point_offsets is not None and not point_offsets.is_cuda):
            raise RuntimeError("MaskedPointToVoxel: points and point_offsets must be CUDA tensors")
        if points.dim() != 2 or points.shape[1] != self.num_point_features:
            raise ValueError(f"MaskedPointToVoxel: points must be [P, {self.num_point_features}], got "
                             f"{tuple(points.shape)}")
        batch = 1
        if point_offsets is not None:
            if point_offsets.dtype != torch.int32 or point_offsets.shape != (self.batch_size + 1,):
                raise ValueError(f"MaskedPointToVoxel: point_offsets must be int32 [{self.batch_size + 1}], got "
                                 f"{point_offsets.dtype} {tuple(point_offsets.shape)}")
            point_offsets = point_offsets.contiguous()
            batch = self.batch_size
        lib = _cabi.load()
        pc = points.contiguous().float()
        n = pc.shape[0]
        bound = self.max_num_voxels_total
        stream = torch.cuda.current_stream(pc.device).cuda_stream
        with torch.no_grad():
            pc_voxel_id = torch.empty([n], dtype=torch.int64, device=pc.device)
            ws = torch.empty(lib.spx_point2voxel_bounded_workspace_size(n, batch, bound), dtype=torch.uint8,
                             device=pc.device)
            _cabi.check(lib.spx_point2voxel_bounded(
                pc.data_ptr() if n else None, n, self.num_point_features, self.ndim, 1, self._c_vsize, self._c_grid,
                self._c_range, point_offsets.data_ptr() if point_offsets is not None else None, batch,
                self.max_num_voxels, bound, self.max_num_points_per_voxel, int(bool(empty_mean)),
                self.voxels.data_ptr(), self.indices.data_ptr(), self.num_per_voxel.data_ptr(),
                pc_voxel_id.data_ptr() if n else None, self.num_valid.data_ptr(), self._bound_status.data_ptr(),
                ws.data_ptr(), ws.numel(), stream), "point2voxel_bounded")
        return self.voxels, self.indices, self.num_per_voxel, pc_voxel_id, self.num_valid


class PointVoxelScatter(object):
    """Per-voxel max / mean / sum of point features, in CUDA (``csrc/point_scatter.cu``) with no host read-back: the
    point -> voxel reduction of a dynamic VFE (OpenPCDet's ``DynamicVoxelVFE`` / ``DynamicPillarVFE``), which keeps
    every point of a voxel.

    ``scatter = PointVoxelScatter(pc_voxel_id, num_rows)`` groups the points once: point ``p`` belongs to output row
    ``pc_voxel_id[p]`` (int32 or int64 ``[P]``, e.g. from :class:`MaskedPointToVoxel`, which sets it for every point
    of a kept voxel, including those beyond ``max_num_points_per_voxel``); a point whose id is outside
    ``[0, num_rows)`` (-1, padding, dropped voxels) is dropped.  Every reduction over the same ids then reuses the
    one sort:

    * ``scatter.max(x)``, ``scatter.mean(x)``, ``scatter.sum(x)``: ``[num_rows, C]`` from ``x [P, C]``,
      differentiable in ``x``.  ``sum`` adds a row's points in fp32 in ascending point index and rounds once;
      ``mean`` divides that sum by the count in fp32 and rounds once.  ``max`` returns the value of the first point
      (in point order) that attains the maximum, bit for bit; a NaN counts as the maximum and -0 / +0 tie.  Its
      gradient goes to that one point per row and channel, as ``torch.max(dim)``'s does (not to a thread-timing
      winner, as ``torch_scatter.scatter_max``, nor split between ties, as ``scatter_reduce("amax")``).  The mean's
      gradient is ``dy / count``, the sum's ``dy``.  A row without points gives 0; dropped points get a zero
      gradient.
    * ``scatter.count``: int32 ``[num_rows]``, the number of points of every row (not capped by
      ``max_num_points_per_voxel``).

    No float atomics: results are bit-reproducible and do not depend on dropped points, wherever they sit.  Nothing
    is read back to the host, so a step captures as one CUDA graph.  float32, float16 and bfloat16 features; P and
    ``num_rows`` below 2^31 - 1.  CUDA only.

    A dynamic-VFE front end (``max_num_points_per_voxel`` only caps the ``voxels`` buffer and may be 1)::

        gen = spconv.MaskedPointToVoxel(vsize, coors_range, 4, max_voxels, 1, batch_size)
        voxels, indices, num_per_voxel, pc_voxel_id, num_valid = gen(points, offsets)
        scatter = spconv.PointVoxelScatter(pc_voxel_id, gen.max_num_voxels_total)
        xyz_mean = scatter.mean(points[:, :3])
        f_cluster = points[:, :3] - spconv.gather_features_by_pc_voxel_id(xyz_mean, pc_voxel_id)
        feats = scatter.max(pfn(torch.cat([points, f_cluster], 1)))   # per-point layers, then the voxel max
        x = spconv.SparseConvTensor(feats, indices, gen.grid_size, gen.batch_size)
        x.num_valid = num_valid
    """

    def __init__(self, pc_voxel_id: torch.Tensor, num_rows: int):
        if int(num_rows) < 0 or int(num_rows) >= 2 ** 31 - 1:
            raise ValueError(f"PointVoxelScatter: num_rows {num_rows} not in [0, 2^31 - 2]")
        self.num_rows = int(num_rows)
        self.row32, self.order, self.offsets = ops.point_scatter_group(pc_voxel_id, self.num_rows)
        self.count = self.offsets.diff()

    def _reduce(self, x: torch.Tensor, mode: str) -> torch.Tensor:
        ops._point_scatter_dtype(x)
        ops._require_cuda(x, "features")
        return Fsp.point_scatter(x, self.row32, self.order, self.offsets, self.count, mode)

    def max(self, x: torch.Tensor) -> torch.Tensor:
        return self._reduce(x, "max")

    def mean(self, x: torch.Tensor) -> torch.Tensor:
        return self._reduce(x, "mean")

    def sum(self, x: torch.Tensor) -> torch.Tensor:
        return self._reduce(x, "sum")


class VoxelPointInterpolator(object):
    """Features of a sparse tensor at query points, trilinear or nearest, in CUDA (``csrc/point_interp.cu``) with no
    host read-back: the voxel -> point step of point-voxel networks (SPVCNN / SPVNAS, PVCNN-style point branches;
    torchsparse's ``voxel_to_point``), from a tensor at any stride.

    ``interp = VoxelPointInterpolator(x, pos, batch_ids, mode="trilinear", normalize=True)`` builds the plan once:

    * ``x``: a :class:`SparseConvTensor` (its ``indices``, ``spatial_shape``, ``batch_size`` and ``num_valid``; its
      features are not read).  A row is used when ``r < num_valid`` (every row without it) and its batch index and
      coordinates are in range; of rows with equal coordinates the lowest is used.
    * ``pos [P, ndim]``: positions in ``x``'s index space, in the axis order of ``indices[:, 1:]`` (zyx in 3-D); row
      ``v``'s feature sits at the integer position ``v``.  :func:`grid_positions` computes them from point
      coordinates.  Cast to float32.  ``batch_ids [P]`` int32 or int64.
    * A point is dropped (output 0, no gradient) when its batch id is outside ``[0, batch_size)`` or a component of
      ``pos`` is not finite or lies outside ``[-1, shape_a)``.
    * ``"trilinear"``: the ``K = 2^ndim`` corners ``floor(pos) + {0, 1}`` per axis with the products of ``f`` /
      ``1 - f`` (``f = pos - floor(pos)``) as weights; a corner without a row gets weight 0, and ``normalize=True``
      divides the found weights by their sum ``+ 1e-8`` (torchsparse's ``calc_ti_weights``, so ported SPVCNN
      checkpoints see the same features near empty voxels).  ``"nearest"``: the one corner ``floor(pos) + (f >= 0.5)`` with
      weight 1 when it exists.

    Then ``interp(features)`` gives ``[P, C]`` from ``features [rows, C]`` (``x.features`` or any other tensor on the
    same coordinates: the plan is reused), differentiable in ``features``.  The forward adds the corners in ascending
    order in fp32 and rounds once; the backward is a weighted sum per row over its points in ascending order.  No
    float atomics: results are bit-reproducible and independent of padding rows and dropped points.  Nothing is read
    back to the host, so a step from raw points to a per-point loss captures as one CUDA graph.
    ``interp.index`` (int32, -1 = no corner) and ``interp.weight`` (fp32) are the ``[P, K]`` table.  float32, float16
    and bfloat16 features; rows, P and P * K below 2^31 - 1.  CUDA only.

    An SPVCNN-style step (point features -> voxels -> convs -> back to the points at stride 2)::

        gen = spconv.MaskedPointToVoxel(vsize, coors_range, 4, max_voxels, 1, batch_size)
        voxels, indices, _, pc_voxel_id, num_valid = gen(points, point_offsets)
        scatter = spconv.PointVoxelScatter(pc_voxel_id, gen.max_num_voxels_total)
        x = spconv.SparseConvTensor(scatter.mean(point_feats), indices, gen.grid_size, batch_size)
        x.num_valid = num_valid
        y = net(x)                                             # e.g. SubMConv3d, then SparseConv3d(k3, s2, p1)
        # batch ids from the offsets, on the device (no sync): point p belongs to sample b when off[b] <= p < off[b+1]
        p = torch.arange(points.shape[0], device=points.device, dtype=torch.int32)
        batch_ids = torch.searchsorted(point_offsets, p, right=True).int() - 1   # -1 / batch_size for padding
        pos = spconv.grid_positions(points[:, :3], vsize, coors_range, stride=2)          # k3 s2 p1: center 0
        interp = spconv.VoxelPointInterpolator(y, pos, batch_ids)
        point_feats = point_mlp(point_feats) + interp(y.features)
    """

    def __init__(self, x, pos: torch.Tensor, batch_ids: torch.Tensor, mode: str = "trilinear", normalize: bool = True):
        if mode not in ops.POINT_INTERP_MODES:
            raise ValueError(f"VoxelPointInterpolator: mode must be 'trilinear' or 'nearest', got {mode!r}")
        self.mode = mode
        self.normalize = bool(normalize)
        self.num_rows = int(x.indices.shape[0])
        nv = getattr(x, "num_valid", None)
        if nv is not None:
            nv = nv.to(device=x.indices.device, dtype=torch.int32).reshape(1)
        self.index, self.weight, self.order, self.offsets = ops.point_interp_plan(
            x.indices, list(x.spatial_shape), int(x.batch_size), nv, pos, batch_ids, mode, normalize)

    def __call__(self, features: torch.Tensor) -> torch.Tensor:
        ops._point_interp_dtype(features)
        ops._require_cuda(features, "features")
        if features.dim() != 2 or features.shape[0] != self.num_rows:
            raise ValueError(f"VoxelPointInterpolator: features must be [{self.num_rows}, C], got "
                             f"{tuple(features.shape)}")
        return Fsp.point_interp(features, self.index, self.weight, self.order, self.offsets)


def _per_axis(v, nd: int, what: str) -> List[float]:
    vals = [float(e) for e in v] if isinstance(v, (list, tuple)) else [float(v)] * nd
    if len(vals) != nd:
        raise ValueError(f"grid_positions: {what} needs {nd} values (xyz order), got {len(vals)}")
    return vals


def grid_positions(points_xyz: torch.Tensor, vsize_xyz: List[float], coors_range_xyz: List[float],
                   stride: Union[int, List[int]] = 1, center: Union[float, List[float]] = 0.0) -> torch.Tensor:
    """Positions ``[P, ndim]`` (fp32, zyx) of points in the index space of a tensor at ``stride`` over the grid of
    :class:`MaskedPointToVoxel` (``vsize_xyz``, ``coors_range_xyz``), for :class:`VoxelPointInterpolator`:
    ``pos_a = ((p_a - lo_a) / vsize_a - 0.5 - center_a) / stride_a``, then the axes reversed (xyz -> zyx).
    ``points_xyz [P, >= ndim]`` (the first ndim columns are used); ``stride`` and ``center`` are one value or one per
    axis (xyz).  A voxel's centre lands on its index at stride 1.  ``center`` is where output ``o`` of the strided
    tensor sits, in input voxels past ``o * stride``:

    ====================================================  ================
    tensor                                                 ``center``
    ====================================================  ================
    the voxelisation grid, or chains of k3 s2 p1 convs     ``0``
    chains of k = s, p = 0 convs (and pools)               ``(s - 1) / 2``
    torchsparse's convention (voxel at its lower corner)   ``-0.5``
    ====================================================  ================
    """
    nd = len(vsize_xyz)
    if len(coors_range_xyz) != 2 * nd:
        raise ValueError(f"grid_positions: coors_range_xyz needs {2 * nd} values, got {len(coors_range_xyz)}")
    if points_xyz.dim() != 2 or points_xyz.shape[1] < nd:
        raise ValueError(f"grid_positions: points must be [P, >= {nd}], got {tuple(points_xyz.shape)}")
    # the per-axis constants are filled on the device (no host -> device copy, so a captured step may call this),
    # and divided by as tensors: a division by a host scalar would become a multiplication by its reciprocal
    k = torch.empty((4, nd), dtype=torch.float32, device=points_xyz.device)
    for i, vals in enumerate(([float(v) for v in coors_range_xyz[:nd]], [float(v) for v in vsize_xyz],
                              _per_axis(center, nd, "center"), _per_axis(stride, nd, "stride"))):
        for a, v in enumerate(vals):
            k[i, a].fill_(v)
    pos = ((points_xyz[:, :nd].float() - k[0]) / k[1] - 0.5 - k[2]) / k[3]
    return pos.flip(1).contiguous()


def gather_features_by_pc_voxel_id(seg_res_features: torch.Tensor, pc_voxel_id: torch.Tensor,
                                   invalid_value: Union[int, float] = 0):
    """Per-point features from per-voxel results (``utils.py:160-176``); points without a voxel get
    ``invalid_value``.  No host synchronisation (a ``where`` over a clamped gather instead of ``nonzero``)."""
    if seg_res_features.device != pc_voxel_id.device:
        pc_voxel_id = pc_voxel_id.to(seg_res_features.device)
    shape = (pc_voxel_id.shape[0], *seg_res_features.shape[1:])
    fill = torch.full(shape, invalid_value, dtype=seg_res_features.dtype, device=seg_res_features.device)
    if seg_res_features.shape[0] == 0:           # no voxels: every id is -1 (nothing to gather from)
        return fill
    valid = pc_voxel_id != -1
    picked = seg_res_features.index_select(0, torch.where(valid, pc_voxel_id, 0))
    return torch.where(valid.view(-1, *([1] * (len(shape) - 1))), picked, fill)
