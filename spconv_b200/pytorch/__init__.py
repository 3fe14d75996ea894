"""``import spconv_b200.pytorch as spconv`` -- the ``spconv.pytorch`` surface of the hot path."""
from ..core import Activation, AlgoHint, ConvAlgo  # noqa: F401
from . import functional, ops  # noqa: F401
from .conv import (SparseConv1d, SparseConv2d, SparseConv3d, SparseConv4d,  # noqa: F401
                   SparseConvolution, SparseConvTranspose1d, SparseConvTranspose2d,
                   SparseConvTranspose3d, SparseConvTranspose4d, SparseInverseConv1d,
                   SparseInverseConv2d, SparseInverseConv3d, SparseInverseConv4d, SubMConv1d,
                   SubMConv2d, SubMConv3d, SubMConv4d)
from .identity import Identity  # noqa: F401
from .core import (CUDAKernelTimer, ImplicitGemmIndiceData, IndiceData,  # noqa: F401
                   SparseConvTensor, scatter_nd)
from .modules import (MaskedBatchNorm1d, MaskedGroupNorm, MaskedSyncBatchNorm1d, RemoveGrid,  # noqa: F401
                      SparseBatchNorm, SparseIdentity, SparseModule, SparseReLU, SparseSequential, SparseSyncBatchNorm, ToDense,
                      assign_name_for_sparse_modules)
from .pool import (MaskedGlobalAvgPool, MaskedGlobalMaxPool, SparseAvgPool1d,  # noqa: F401
                   SparseAvgPool2d, SparseAvgPool3d, SparseGlobalAvgPool, SparseGlobalMaxPool, SparseMaxPool1d,
                   SparseMaxPool2d, SparseMaxPool3d, SparseMaxPool4d)
from .tables import (AddTable, ConcatTable, JoinTable, MaskedAddTable, MaskedAddTableMisaligned,  # noqa: F401
                     MaskedJoinTable)
from .spatial import MaskedRemoveDuplicate  # noqa: F401
from .utils_fuse import (fuse_act, fuse_bn, fuse_bn_act_sequential, fuse_bn_weights)  # noqa: F401
from . import quantized  # noqa: F401
from .fp8 import (Fp8SparseConv, calibrate_fp8_output_scale, convert_to_fp8, dequantize_fp8,  # noqa: F401
                  quantize_fp8, quantize_fp8_weight)
from .graph import GraphedStep, graph_capture  # noqa: F401
from .utils import (MaskedPointToVoxel, PointToVoxel, PointVoxelScatter, VoxelPointInterpolator,  # noqa: F401
                    gather_features_by_pc_voxel_id, grid_positions)
from .prefetch import RulebookPrefetcher  # noqa: F401
from .bounds import check_bounds, set_output_bounds  # noqa: F401
