"""MaskedSyncBatchNorm1d, the parts that need no GPU: the C descriptor's layout, argument validation of the
C entry points and of the Python transport before any launch, which modules convert_masked_sync_batchnorm
replaces, state_dict compatibility with nn.SyncBatchNorm, the eval-mode path (torch's row-wise batch_norm),
and SparseSyncBatchNorm's refusal of padded training input."""
import copy
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch
from torch import nn

from tests.test_masked_batchnorm_cpu import _backbone, _tensor

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedBatchNorm1d, MaskedSyncBatchNorm1d, SparseSyncBatchNorm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ("fwd_local", "fwd_merge", "bwd_local", "bwd_merge")


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def test_descriptor_layout_matches_the_header(tmp_path):
    """spx_masked_sync_bn has the same size and field offsets in ctypes as in C"""
    from spconv_b200 import _cabi
    cls = _cabi.MaskedSyncBN
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "spconv_b200.h"', "int main(void) {",
             '  printf("size %zu\\n", sizeof(spx_masked_sync_bn));']
    lines += [f'  printf("{f} %zu\\n", offsetof(spx_masked_sync_bn, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = dict(ln.split() for ln in subprocess.run([str(exe)], capture_output=True, text=True,
                                                   check=True).stdout.split("\n") if ln.strip())
    assert int(out.pop("size")) == ctypes.sizeof(cls)
    assert {f: int(v) for f, v in out.items()} == {f: getattr(cls, f).offset for f, _ in cls._fields_}


def test_every_pointer_of_the_new_entry_points_is_covered():
    """every pointer field of the descriptor and of spx_peer_allgather is misaligned by
    test_masked_sync_batchnorm_gpu.py::test_misaligned_operands_give_the_same_bits or explained here"""
    from spconv_b200 import _cabi
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "spconv_b200.h")).read(), flags=re.S)
    body = re.search(r"typedef struct spx_masked_sync_bn \{(.*?)\} spx_masked_sync_bn;", text, re.S).group(1)
    ptrs = set()
    for decl in body.split(";"):
        if "*" in decl:
            ptrs |= {p.strip().lstrip("*").strip() for p in decl.split("*", 1)[1].split(",")}
    assert ptrs == {f for f, t in _cabi.MaskedSyncBN._fields_ if t is ctypes.c_void_p}
    swept = {"x", "dy"}
    explained = {
        "y": "output allocated by the library", "dx": "output allocated by the library",
        "num_valid": "one int32 read with __ldg",
        "weight": "a per-channel vector read element by element", "bias": "a per-channel vector read element by element",
        "running_mean": "a per-channel vector read and written element by element",
        "running_var": "a per-channel vector read and written element by element",
        "num_batches_tracked": "one int64 read", "save_mean": "output allocated by the library",
        "save_invstd": "output allocated by the library", "dweight": "output allocated by the library",
        "dbias": "output allocated by the library", "local": "fp32 vector allocated by the library",
        "gathered": "fp32 matrix allocated by the library",
    }
    assert ptrs == swept | set(explained)
    gather = re.search(r"int\s+spx_peer_allgather\s*\(([^;]*)\)\s*;", text, re.S).group(1)
    assert [p.split("*")[-1].strip() for p in gather.split(",") if "*" in p] == ["pg", "src", "dst"]
    # src / dst: 32-bit words read and written one at a time (peer_push_kernel, peer_finish_kernel)


def test_workspace_size(lib):
    fn = lib.spx_masked_sync_bn_workspace_size
    for rows in (0, 1, 512, 513, 100_000):
        assert fn(rows, 64) == lib.spx_masked_bn_fwd_train_workspace_size(rows, 64)
    assert fn(-1, 16) == 0 and fn(10, 0) == 0


def test_entry_points_validate_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import ctypes, sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def desc(**kw):",
        "    d = _cabi.MaskedSyncBN()",
        "    d.rows, d.channels, d.dtype, d.param_dtype, d.world, d.eps, d.momentum = 10, 16, 1, 0, 2, 1e-5, 0.1",
        "    for f in ('x', 'y', 'dy', 'dx', 'weight', 'bias', 'running_mean', 'running_var', 'num_batches_tracked',",
        "              'save_mean', 'save_invstd', 'dweight', 'dbias', 'local', 'gathered'):",
        "        setattr(d, f, P)",
        "    for k, v in kw.items():",
        "        setattr(d, k, v)",
        "    return d",
        "def call(name, ws=P, wsb=1 << 30, **kw):",
        "    return getattr(lib, 'spx_masked_sync_bn_' + name)(ctypes.byref(desc(**kw)), ws, wsb, None)",
        "def expect(rc, text):",
        "    assert rc == 2 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        f"for n in {ENTRY_POINTS!r}:",
        "    expect(getattr(lib, 'spx_masked_sync_bn_' + n)(None, P, 1 << 30, None), 'descriptor is NULL')",
        "    expect(call(n, rows=-1), 'bad row count')",
        "    expect(call(n, rows=(1 << 24) + 1), 'at most 2^24')",
        "    expect(call(n, channels=0), 'channels must be')",
        "    expect(call(n, dtype=3), 'unsupported dtype')",
        "    expect(call(n, param_dtype=2), 'parameter dtype')",
        "    expect(call(n, ws=None), 'NULL pointer')",
        "    expect(call(n, wsb=64), 'workspace too small')",
        "    expect(call(n, x=None), 'NULL pointer')",
        "for n in ('fwd_local', 'bwd_local'):",
        "    expect(call(n, local=None), 'NULL pointer')",
        "for n in ('fwd_merge', 'bwd_merge'):",
        "    expect(call(n, gathered=None), 'NULL pointer')",
        "    expect(call(n, world=0), 'world 0 out of range')",
        "    expect(call(n, world=17), 'world 17 out of range')",
        "for n in ('fwd_merge', 'bwd_local', 'bwd_merge'):",
        "    expect(call(n, save_mean=None), 'NULL pointer')",
        "expect(call('fwd_merge', y=None), 'NULL pointer')",
        "expect(call('fwd_merge', running_var=None), 'both be given')",
        "expect(call('fwd_merge', cumulative=1, num_batches_tracked=None), 'needs num_batches_tracked')",
        "expect(call('fwd_merge', eps=0.0), 'eps must be positive')",
        "expect(call('bwd_local', dy=None), 'NULL pointer')",
        "expect(call('bwd_merge', dx=None), 'NULL pointer')",
        "g = _cabi.PeerGroup()",
        "g.world, g.rank, g.capacity_bytes = 2, 2, 1 << 10",
        "expect(lib.spx_peer_allgather(ctypes.byref(g), P, 16, P, None), 'bad peer group')",
        "g.rank = 1",
        "expect(lib.spx_peer_allgather(ctypes.byref(g), P, 257, P, None), 'exceed the exchange capacity')",
        "expect(lib.spx_peer_allgather(ctypes.byref(g), P, 16, P, None), 'buffer of rank 0 is NULL')",
        "expect(lib.spx_peer_allgather(ctypes.byref(g), None, 16, P, None), 'NULL src or dst')",
        "expect(lib.spx_peer_allgather(None, P, 16, P, None), 'peer group is NULL')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


class _FakePeers:
    """the attributes of a PeerGroup the transport reads, without a device buffer"""

    def __init__(self, world, rank=0, capacity=8 << 20):
        from spconv_b200 import _cabi
        self.world, self.rank = world, rank
        self.group = _cabi.PeerGroup()
        self.group.world, self.group.rank, self.group.capacity_bytes = world, rank, capacity


@pytest.fixture
def single_process_group():
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=0, world_size=1, store=dist.HashStore())
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


def test_transport_choice_and_host_checks(single_process_group):
    from spconv_b200.pytorch import ops
    assert ops.sync_bn_transport().kind == "local"                       # torch.distributed with one rank
    assert ops.sync_bn_transport(single_process_group).kind == "local"
    try:
        ops.set_peer_group(_FakePeers(2))
        t = ops.sync_bn_transport()
        assert (t.kind, t.world) == ("peer", 2)
        with pytest.raises(RuntimeError, match="process_group has 1 ranks, the installed peer group 2"):
            ops.sync_bn_transport(single_process_group)
        ops.set_peer_group(_FakePeers(1))
        assert ops.sync_bn_transport(single_process_group).kind == "peer"
        x = torch.empty((100, 64), device="meta")
        ops._sync_bn_check(x, ops.sync_bn_transport())
        with pytest.raises(RuntimeError, match="at most 2"):
            ops._sync_bn_check(torch.empty(((1 << 24) + 1, 4), device="meta"), ops.sync_bn_transport())
        ops.set_peer_group(_FakePeers(2, capacity=256))
        with pytest.raises(RuntimeError, match="exceed the peer group's exchange capacity"):
            ops._sync_bn_check(x, ops.sync_bn_transport())
        ops._sync_bn_check(torch.empty((5, 31), device="meta"), ops.sync_bn_transport())     # 63 values fit
        ops.set_peer_group(_FakePeers(2, rank=2))
        with pytest.raises(RuntimeError, match="bad peer group"):
            ops._sync_bn_check(x, ops.sync_bn_transport())
    finally:
        ops.set_peer_group(None)


def _sync_backbone():
    net = _backbone()
    net["enc"][3].add_module("5", MaskedBatchNorm1d(8))
    net["enc"].add_module("5", SparseSyncBatchNorm(8, momentum=0.3))
    return net


def test_convert_masked_sync_batchnorm_selects_the_right_modules():
    net = _sync_backbone()
    before = copy.deepcopy(net.state_dict())
    params = {n: p for n, p in net.named_parameters()}
    group = object()
    out = MaskedSyncBatchNorm1d.convert_masked_sync_batchnorm(net, process_group=group)
    assert out is net
    enc = net["enc"]
    assert type(enc[1]) is MaskedSyncBatchNorm1d and enc[1].momentum is None
    inner = enc[3]
    assert type(inner[1]) is MaskedSyncBatchNorm1d and not inner[1].affine
    assert type(inner[3]) is MaskedSyncBatchNorm1d                     # nn.SyncBatchNorm
    assert type(inner[4].inner) is MaskedSyncBatchNorm1d
    assert type(inner[5]) is MaskedSyncBatchNorm1d                     # MaskedBatchNorm1d
    assert type(enc[4].inner) is MaskedSyncBatchNorm1d and not enc[4].inner.track_running_stats
    assert enc[4].inner.running_mean is None and enc[4].inner.num_batches_tracked is None
    assert type(enc[5].inner) is MaskedSyncBatchNorm1d and enc[5].inner.momentum == 0.3
    assert all(m.process_group is group for m in net.modules() if isinstance(m, MaskedSyncBatchNorm1d))
    assert type(net["head"][1]) is nn.BatchNorm1d
    for n, p in net.named_parameters():
        assert p is params[n], n
    after = net.state_dict()
    assert list(after) == list(before)
    for k in before:
        assert torch.equal(after[k], before[k]), k
    net2 = _sync_backbone().eval()
    MaskedSyncBatchNorm1d.convert_masked_sync_batchnorm(net2)
    assert not net2["enc"][1].training and net2["enc"][1].process_group is None
    sbn = nn.SyncBatchNorm(8, process_group=group)
    conv = MaskedSyncBatchNorm1d.convert_masked_sync_batchnorm(spconv.SparseSequential(sbn))
    assert conv[0].process_group is group                             # a SyncBatchNorm keeps its own group
    bn = nn.BatchNorm1d(3)
    assert MaskedSyncBatchNorm1d.convert_masked_sync_batchnorm(bn) is bn and type(bn) is nn.BatchNorm1d


def test_convert_masked_batchnorm_is_unchanged():
    """convert_masked_batchnorm still skips SyncBatchNorm, SparseSyncBatchNorm and the sync module"""
    net = MaskedSyncBatchNorm1d.convert_masked_sync_batchnorm(_sync_backbone())
    kinds = [type(m) for m in net.modules()]
    MaskedBatchNorm1d.convert_masked_batchnorm(net)
    assert [type(m) for m in net.modules()] == kinds
    seq = spconv.SparseSequential(nn.SyncBatchNorm(4), SparseSyncBatchNorm(4))
    MaskedBatchNorm1d.convert_masked_batchnorm(seq)
    assert type(seq[0]) is nn.SyncBatchNorm and type(seq[1].inner) is nn.SyncBatchNorm


def test_state_dict_loads_both_ways_with_sync_batchnorm():
    m = MaskedSyncBatchNorm1d(5)
    ref = nn.SyncBatchNorm(5)
    assert list(m.state_dict()) == list(ref.state_dict())
    assert [n for n, _ in m.named_parameters()] == [n for n, _ in ref.named_parameters()]
    assert [n for n, _ in m.named_buffers()] == [n for n, _ in ref.named_buffers()]
    with torch.no_grad():
        ref.weight.uniform_(0.5, 1.5)
        ref.running_var.uniform_(0.5, 2)
        ref.num_batches_tracked.fill_(9)
    m.load_state_dict(ref.state_dict())
    for k, v in ref.state_dict().items():
        assert torch.equal(m.state_dict()[k], v), k
    with torch.no_grad():
        m.bias.fill_(0.5)
        m.running_mean.fill_(-0.25)
    back = nn.SyncBatchNorm(5)
    back.load_state_dict(m.state_dict())
    for k, v in m.state_dict().items():
        assert torch.equal(back.state_dict()[k], v), k
    plain = _sync_backbone()
    conv = MaskedSyncBatchNorm1d.convert_masked_sync_batchnorm(_sync_backbone())
    assert list(plain.state_dict()) == list(conv.state_dict())
    conv.load_state_dict(plain.state_dict())


def test_eval_mode_is_torch_batch_norm_row_wise():
    x = _tensor()
    bn = nn.SyncBatchNorm(8)
    with torch.no_grad():
        bn.running_mean.uniform_(-1, 1)
        bn.running_var.uniform_(0.5, 2)
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-1, 1)
    bn.eval()
    seq = MaskedSyncBatchNorm1d.convert_masked_sync_batchnorm(spconv.SparseSequential(copy.deepcopy(bn)))
    assert type(seq[0]) is MaskedSyncBatchNorm1d and not seq[0].training
    want = nn.functional.batch_norm(x.features, bn.running_mean, bn.running_var, bn.weight, bn.bias, False, 0.0,
                                    bn.eps)
    assert torch.equal(seq(x).features, want)
    p = x.pad_to(9)
    y = seq(p)
    assert y.num_valid is p.num_valid and torch.equal(y.features[:6], want)
    empty = spconv.SparseConvTensor(torch.zeros((0, 8)), torch.zeros((0, 4), dtype=torch.int32), [6, 6, 6], 1)
    assert seq(empty) is empty
    with pytest.raises(ValueError, match="features of shape"):
        MaskedSyncBatchNorm1d(4).eval()(x)
    with pytest.raises(ValueError, match="features of shape"):
        MaskedSyncBatchNorm1d(4)(x)


def test_sparse_sync_batchnorm_refuses_padded_training_input():
    p = _tensor(5).pad_to(8)
    m = SparseSyncBatchNorm(8)
    assert type(m.inner) is nn.SyncBatchNorm
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        m(p)
    m.eval()
    with torch.no_grad():
        m.inner.running_var.fill_(2.0)
    y = m(p)                                               # eval is row-wise: padding is allowed
    assert torch.equal(y.features, m.inner(p.features))
