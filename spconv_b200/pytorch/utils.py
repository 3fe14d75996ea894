"""Point cloud -> voxel front end (``spconv/pytorch/utils.py:23-176``): ``PointToVoxel`` and
``gather_features_by_pc_voxel_id``, plus ``MaskedPointToVoxel`` and ``PointVoxelScatter``.  CUDA only; the
kernels live in ``csrc/pointops.cu`` and ``csrc/point_scatter.cu``.

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
