"""Flags of the reference that touch the hot path (``spconv/constants.py``)."""
import os

# spconv/constants.py:37-42 -- weights are always KRSC in this engine
SAVED_WEIGHT_LAYOUT = os.getenv("SPCONV_SAVED_WEIGHT_LAYOUT", "")
if SAVED_WEIGHT_LAYOUT != "":
    assert SAVED_WEIGHT_LAYOUT in ["KRSC", "RSKC", "RSCK"], \
        "please set SAVED_WEIGHT_LAYOUT to KRSC, RSKC or RSCK"
ALL_WEIGHT_IS_KRSC = True
# spconv/constants.py:117 -- fp32 tensors multiply in exact fp32 unless TF32 is allowed
SPCONV_ALLOW_TF32 = os.getenv("SPCONV_ALLOW_TF32", "0") == "1"
# spconv/constants.py:121
SPCONV_DO_SORT = os.getenv("SPCONV_DO_SORT", "1") == "1"
SPCONV_DEBUG_SAVE_PATH = os.getenv("SPCONV_DEBUG_SAVE_PATH", "")
SPCONV_FX_TRACE_MODE = os.getenv("SPCONV_FX_TRACE_MODE", "0") == "1"


class AllocKeys:
    """Named buffers of the reference allocator protocol (``spconv/constants.py:66-98``); kept
    as documentation of which tensor is which, the C ABI takes plain pointers."""
    PairFwd = "PairFwd"
    PairBwd = "PairBwd"
    IndiceNumPerLoc = "IndiceNumPerLoc"
    OutIndices = "OutIndices"
    PairMask = "PairMask"
    PairMaskBwd = "PairMaskBwd"
    MaskArgSort = "MaskArgSort"
    MaskArgSortBwd = "MaskArgSortBwd"
    MaskOutputFwd = "MaskOutputFwd"
    OutFeatures = "OutFeatures"
    DIn = "DIn"
    DFilters = "DFilters"
