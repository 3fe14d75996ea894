"""Point cloud -> voxel front end (``spconv/pytorch/utils.py:23-176``): ``PointToVoxel`` and
``gather_features_by_pc_voxel_id``.  CUDA only; the kernels live in ``csrc/pointops.cu``.

Unlike the reference's GPU generator (atomic appends: voxel order and the points kept per voxel
depend on scheduling) the result is deterministic and equal to the reference's CPU generator
(``Point2VoxelCPU``, ``spconv/csrc/sparse/pointops.py:589-695``): voxels are numbered by their first
point, a voxel keeps its first ``max_num_points_per_voxel`` points, both in input order.  A point is
in a voxel when ``floor((p - lo) / vsize)`` (fp32) is a finite value in ``[0, grid)`` on every axis; a
point with a NaN or infinite coordinate gets ``pc_voxel_id`` -1 and makes no voxel.
"""
from __future__ import annotations

import ctypes
from typing import List, Union

import numpy as np
import torch

from .. import _cabi


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


def gather_features_by_pc_voxel_id(seg_res_features: torch.Tensor, pc_voxel_id: torch.Tensor,
                                   invalid_value: Union[int, float] = 0):
    """Per-point features from per-voxel results (``utils.py:160-176``); points without a voxel get
    ``invalid_value``."""
    if seg_res_features.device != pc_voxel_id.device:
        pc_voxel_id = pc_voxel_id.to(seg_res_features.device)
    shape = (pc_voxel_id.shape[0], *seg_res_features.shape[1:])
    res = torch.full(shape, invalid_value, dtype=seg_res_features.dtype, device=seg_res_features.device)
    valid = torch.nonzero(pc_voxel_id != -1).view(-1)
    res[valid] = seg_res_features[pc_voxel_id[valid]]
    return res
