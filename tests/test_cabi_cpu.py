"""The C-ABI library builds, loads without a GPU and exports exactly what include/spconv_b200.h
declares (no compute calls here)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def _header_functions():
    text = open(os.path.join(ROOT, "include", "spconv_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(spx_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported_and_bound(lib):
    from spconv_b200 import _cabi
    declared = _header_functions()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in the header but missing from the .so"
        assert name in _cabi.SIGNATURES, f"{name} has no ctypes signature"
    assert sorted(_cabi.SIGNATURES) == declared


def test_no_torch_or_python_dependency():
    """plain C ABI: the library must not link libtorch / libpython / libcuda.so"""
    import subprocess
    from spconv_b200 import _cabi
    out = subprocess.run(["ldd", _cabi.LIB_PATH], capture_output=True, text=True).stdout
    for forbidden in ("libtorch", "libpython", "libc10", "libcuda.so"):
        assert forbidden not in out, out


def test_host_only_entry_points(lib):
    import ctypes
    from spconv_b200 import _cabi
    assert lib.spx_version() >= 100
    g = _cabi.make_geometry(3, 1, [41, 1600, 1408], [21, 800, 704], [3] * 3, [2] * 3, [1] * 3, [1] * 3)
    # get_handcrafted_max_act_out (all.py:1559-1580): N * prod(ceil(k/s)) capped by kv*N
    assert lib.spx_conv_max_out(ctypes.byref(g), 1000) == 8000
    g2 = _cabi.make_geometry(3, 1, [8] * 3, [8] * 3, [3] * 3, [1] * 3, [1] * 3, [1] * 3)
    assert lib.spx_conv_max_out(ctypes.byref(g2), 10) == 270
    assert lib.spx_rulebook_workspace_size(ctypes.byref(g), 100000, 0, 0) > 100000 * 8 * 8
    assert lib.spx_rulebook_workspace_size(ctypes.byref(g), 100000, 0, 1) >= 2 * 100000 * 8
    assert lib.spx_mask_argsort_workspace_size(100000, 1) > 100000 * 4 * 4
    assert lib.spx_native_pairs_workspace_size(100000, 27) > 0
    # The launch counter and the last kernel family are process-wide, and GPU tests may have run in this
    # process before: check in a fresh process that the host entry points launch nothing.
    import subprocess
    import sys
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "g = _cabi.make_geometry(3, 1, [41, 1600, 1408], [21, 800, 704], [3] * 3, [2] * 3, [1] * 3, [1] * 3)",
        "lib.spx_version()",
        "lib.spx_conv_max_out(ctypes.byref(g), 1000)",
        "lib.spx_rulebook_workspace_size(ctypes.byref(g), 100000, 0, 0)",
        "lib.spx_rulebook_workspace_size(ctypes.byref(g), 100000, 0, 1)",
        "lib.spx_mask_argsort_workspace_size(100000, 1)",
        "lib.spx_native_pairs_workspace_size(100000, 27)",
        "print(lib.spx_launch_count(1), lib.spx_last_kernel_family())",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0", "0"], res.stdout


def test_argument_validation_reports_errors(lib):
    """invalid arguments fail before touching the device and leave a message (TV_ASSERT_RT_ERR role)"""
    import ctypes
    from spconv_b200 import _cabi
    bad = _cabi.make_geometry(3, 1, [8] * 3, [8] * 3, [2] * 3, [1] * 3, [0] * 3, [1] * 3)
    rc = lib.spx_subm_rulebook(ctypes.byref(bad), 1, 10, 1, None, None, 1, 1, None)
    assert rc != 0 and "odd ksize" in _cabi.last_error()
    bad.ndim = 7
    rc = lib.spx_subm_rulebook(ctypes.byref(bad), 1, 10, 1, None, None, 1, 1, None)
    assert rc != 0 and "ndim" in _cabi.last_error()
    d = _cabi.GemmDesc()
    d.kv, d.c_in, d.c_out, d.dtype = 0, 16, 16, _cabi.SPX_F16
    assert lib.spx_implicit_gemm_fwd(ctypes.byref(d), None, None, None, None, 0, 0.0, None) != 0
    assert "kernel volume" in _cabi.last_error()
    with pytest.raises(RuntimeError, match="kernel volume"):
        _cabi.check(2, "x")


def test_debug_configure_accepts_only_the_tf32_switches(lib):
    """spx_debug_configure takes debug bits 256 and 4096 only: any other bit, and any trace buffer, is
    refused before a CUDA call, so an A/B run of a path the library no longer has fails loudly"""
    import ctypes
    from spconv_b200 import _cabi
    try:
        for bits in (1, 2, 4, 8, 16, 64, 128, 512, 1024, 2048, 8192, 16384, 256 | 64):
            assert lib.spx_debug_configure(-1, 0, bits, None, 0) == 2, bits
            msg = _cabi.last_error()
            assert "debug_bits" in msg and "256" in msg and "4096" in msg, msg
        for bits in (256, 4096, 256 | 4096, 0):
            assert lib.spx_debug_configure(-1, 0, bits, None, 0) == 0, bits
        assert lib.spx_debug_configure(-1, 0, 0, ctypes.c_void_p(1 << 20), 8 * 2048 * 8) == 2
        assert "trace buffer" in _cabi.last_error()
    finally:
        _cabi.check(lib.spx_debug_configure(-1, 0, 0, None, 0), "debug_configure")


def test_tile_table_elems_formula_matches_the_library():
    """ops._tile_tables sizes the table buffer without a native call; the formula must stay equal to
    spx_tile_table_elems (layout documented in include/spconv_b200.h)"""
    from spconv_b200 import _cabi
    lib = _cabi.load()
    for rows in (1, 127, 128, 129, 100_000, 1_234_567):
        for kv in (1, 8, 27, 81, 128):
            tiles = max((rows + 127) // 128, 1)
            assert lib.spx_tile_table_elems(rows, kv) == tiles * (kv + 1) * 128 + tiles * 8 + 64


def test_ctypes_structs_match_the_header_layout(tmp_path):
    """the three structs that cross the boundary have the same size and field offsets in ctypes as in C
    (include/spconv_b200.h compiled by gcc) -- a silent mismatch would shift every pointer argument"""
    import ctypes
    import subprocess
    from spconv_b200 import _cabi
    structs = {"spx_conv_geometry": _cabi.ConvGeometry, "spx_gemm_desc": _cabi.GemmDesc, "spx_peer_group": _cabi.PeerGroup}
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "spconv_b200.h"', "int main(void) {"]
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    seen = 0
    for ln in out:
        if not ln.strip():
            continue
        cname, field, val = ln.split()
        cls = structs[cname]
        want = ctypes.sizeof(cls) if field == "size" else getattr(cls, field).offset
        assert int(val) == want, f"{cname}.{field}: C {val} vs ctypes {want}"
        seen += 1
    assert seen == sum(len(c._fields_) + 1 for c in structs.values())


def test_peer_exchange_host_side_validation(lib):
    """spx_peer_* argument checks and sizes run without a GPU (no buffer is created here)"""
    import ctypes
    from spconv_b200 import _cabi
    assert _cabi.SPX_MAX_PEERS == 16
    # two epochs of this rank's own fp32 slices + the 4 KB header (state, flags)
    assert lib.spx_peer_buffer_bytes(1 << 20, 8) == 4096 + 2 * (1 << 20)
    assert lib.spx_peer_buffer_bytes(1 << 20, 0) == 0 and lib.spx_peer_buffer_bytes(1 << 20, 17) == 0
    g = _cabi.PeerGroup()
    g.world, g.rank, g.capacity_bytes = 2, 5, 1 << 20
    assert lib.spx_peer_push(ctypes.byref(g), 1, 16, _cabi.SPX_F32, None) != 0
    assert "bad peer group" in _cabi.last_error()
    g.rank = 1
    assert lib.spx_peer_finish(ctypes.byref(g), 1, (1 << 20), _cabi.SPX_F32, 1.0, None) != 0
    assert "exceed the exchange capacity" in _cabi.last_error()
    assert lib.spx_peer_push(ctypes.byref(g), 1, 16, _cabi.SPX_F32, None) != 0
    assert "buffer of rank 0 is NULL" in _cabi.last_error()
    d = _cabi.GemmDesc()
    d.kv, d.c_in, d.c_out, d.dtype, d.n_in, d.n_out = 27, 16, 16, _cabi.SPX_F16, 10, 10
    assert lib.spx_implicit_gemm_wgrad_push(ctypes.byref(d), 1, 1, 1, None, 0, None, None) != 0
    assert "peer group is NULL" in _cabi.last_error()
