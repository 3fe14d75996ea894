"""MaskedBatchNorm1d, the parts that need no GPU: argument validation of the C entry points before any launch,
workspace sizes, which modules convert_masked_batchnorm replaces, state_dict compatibility with nn.BatchNorm1d
and the eval-mode path (torch's row-wise batch_norm, which also runs on the CPU)."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch import nn

from tests.util import random_cloud

import spconv_b200.pytorch as spconv
from spconv_b200.pytorch import MaskedBatchNorm1d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from spconv_b200 import _cabi, build
    build.build()
    return _cabi.load()


def test_workspace_sizes(lib):
    for fn in (lib.spx_masked_bn_fwd_train_workspace_size, lib.spx_masked_bn_bwd_workspace_size):
        assert fn(-1, 16) == 0 and fn(100, 0) == 0
        assert fn(0, 16) > 0                               # the per-channel coefficients
        prev = 0
        for rows in (1, 512, 513, 100_000):
            cur = fn(rows, 64)
            assert cur >= prev and cur >= (rows + 511) // 512 * 64 * 8
            prev = cur


def test_entry_points_validate_before_any_launch():
    """run in a fresh process: the launch counter is process-wide"""
    script = "\n".join([
        "import sys",
        f"sys.path.insert(0, {ROOT!r})",
        "from spconv_b200 import _cabi",
        "lib = _cabi.load()",
        "P = 1 << 20",
        "def fwd(x=P, y=P, rows=10, c=16, dt=1, nv=None, w=P, b=P, rm=P, rv=P, nbt=P, pdt=0, mom=0.1, cum=0,",
        "        eps=1e-5, sm=P, si=P, ws=P, wsb=1 << 30):",
        "    return lib.spx_masked_bn_fwd_train(x, y, rows, c, dt, nv, w, b, rm, rv, nbt, pdt, mom, cum, eps, sm, si,",
        "                                       ws, wsb, None)",
        "def bwd(x=P, dy=P, dx=P, rows=10, c=16, dt=1, nv=None, w=P, pdt=0, sm=P, si=P, dw=P, db=P, ws=P,",
        "        wsb=1 << 30):",
        "    return lib.spx_masked_bn_bwd(x, dy, dx, rows, c, dt, nv, w, pdt, sm, si, dw, db, ws, wsb, None)",
        "def expect(rc, text):",
        "    assert rc == 2 and text in _cabi.last_error(), (rc, _cabi.last_error())",
        "for f in (fwd, bwd):",
        "    expect(f(rows=-1), 'bad row count')",
        "    expect(f(c=0), 'channels must be')",
        "    expect(f(dt=3), 'unsupported dtype')",
        "    expect(f(pdt=2), 'parameter dtype')",
        "    expect(f(dt=0, pdt=1), 'parameter dtype')",
        "    expect(f(sm=None), 'NULL pointer')",
        "    expect(f(ws=None), 'NULL pointer')",
        "    expect(f(x=None), 'NULL pointer')",
        "    expect(f(wsb=64), 'workspace too small')",
        "expect(fwd(y=None), 'NULL pointer')",
        "expect(fwd(rm=None), 'both be given')",
        "expect(fwd(rv=None), 'both be given')",
        "expect(fwd(cum=1, nbt=None), 'needs num_batches_tracked')",
        "expect(fwd(eps=0.0), 'eps must be positive')",
        "expect(bwd(dy=None), 'NULL pointer')",
        "expect(bwd(dx=None), 'NULL pointer')",
        "print(lib.spx_launch_count(1))",
    ])
    res = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert res.stdout.split() == ["0"], res.stdout


def _backbone():
    torch.manual_seed(0)
    head = nn.Sequential(nn.Linear(8, 8), nn.BatchNorm1d(8))          # a dense head: left alone
    net = nn.ModuleDict({
        "enc": spconv.SparseSequential(
            spconv.SubMConv3d(4, 8, 3, indice_key="a"), nn.BatchNorm1d(8, momentum=None), nn.ReLU(),
            spconv.SparseSequential(
                spconv.SparseConv3d(8, 8, 3, stride=2), nn.BatchNorm1d(8, affine=False), nn.ReLU(),
                nn.SyncBatchNorm(8), spconv.SparseBatchNorm(8)),
            spconv.SparseBatchNorm(8, track_running_stats=False)),
        "head": head,
    })
    # non-default running stats, so that carried-over buffers are recognisable
    for m in net.modules():
        if isinstance(m, nn.modules.batchnorm._BatchNorm) and m.running_mean is not None:
            m.running_mean.uniform_(-1, 1)
            m.running_var.uniform_(0.5, 2)
            m.num_batches_tracked.fill_(7)
    return net


def test_convert_masked_batchnorm_selects_the_right_modules():
    net = _backbone()
    before = copy.deepcopy(net.state_dict())
    params = {n: p for n, p in net.named_parameters()}
    out = MaskedBatchNorm1d.convert_masked_batchnorm(net)
    assert out is net
    enc = net["enc"]
    assert type(enc[1]) is MaskedBatchNorm1d and enc[1].momentum is None
    inner = enc[3]
    assert type(inner[1]) is MaskedBatchNorm1d and not inner[1].affine
    assert type(inner[3]) is nn.SyncBatchNorm
    assert type(inner[4].inner) is MaskedBatchNorm1d
    assert type(enc[4].inner) is MaskedBatchNorm1d and not enc[4].inner.track_running_stats
    assert enc[4].inner.running_mean is None and enc[4].inner.num_batches_tracked is None
    assert type(net["head"][1]) is nn.BatchNorm1d
    assert type(enc[0]) is spconv.SubMConv3d and type(enc[2]) is nn.ReLU
    # parameters and buffers are carried over as the same objects
    for n, p in net.named_parameters():
        assert p is params[n], n
    after = net.state_dict()
    assert list(after) == list(before)
    for k in before:
        assert torch.equal(after[k], before[k]), k
    assert int(enc[1].num_batches_tracked) == 7
    # training flags follow the replaced module
    net2 = _backbone().eval()
    MaskedBatchNorm1d.convert_masked_batchnorm(net2)
    assert not net2["enc"][1].training
    # a bare BatchNorm1d is not inside a sparse container: unchanged
    bn = nn.BatchNorm1d(3)
    assert MaskedBatchNorm1d.convert_masked_batchnorm(bn) is bn and type(bn) is nn.BatchNorm1d


def test_state_dict_loads_both_ways():
    plain = _backbone()
    conv = MaskedBatchNorm1d.convert_masked_batchnorm(_backbone())
    for m in conv.modules():                               # different values, same keys
        if isinstance(m, nn.modules.batchnorm._BatchNorm) and m.running_mean is not None:
            m.running_mean.fill_(0.25)
            m.num_batches_tracked.fill_(3)
    assert list(plain.state_dict()) == list(conv.state_dict())
    fresh = MaskedBatchNorm1d.convert_masked_batchnorm(_backbone())
    fresh.load_state_dict(plain.state_dict())
    for k, v in plain.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v), k
    back = _backbone()
    back.load_state_dict(conv.state_dict())
    for k, v in conv.state_dict().items():
        assert torch.equal(back.state_dict()[k], v), k
    m = MaskedBatchNorm1d(5)
    ref = nn.BatchNorm1d(5)
    assert list(m.state_dict()) == list(ref.state_dict())
    assert [n for n, _ in m.named_parameters()] == [n for n, _ in ref.named_parameters()]
    assert [n for n, _ in m.named_buffers()] == [n for n, _ in ref.named_buffers()]


def _tensor(n=6, c=8):
    rng = np.random.default_rng(1)
    feats, inds = random_cloud(rng, [6, 6, 6], [n], c)
    return spconv.SparseConvTensor(torch.from_numpy(feats), torch.from_numpy(inds), [6, 6, 6], 1)


def test_eval_mode_is_torch_batch_norm_row_wise():
    x = _tensor()
    bn = nn.BatchNorm1d(8)
    bn.running_mean.uniform_(-1, 1)
    bn.running_var.uniform_(0.5, 2)
    bn.weight.data.uniform_(0.5, 1.5)
    bn.bias.data.uniform_(-1, 1)
    bn.eval()
    seq = MaskedBatchNorm1d.convert_masked_batchnorm(spconv.SparseSequential(copy.deepcopy(bn)))
    assert type(seq[0]) is MaskedBatchNorm1d and not seq[0].training
    assert torch.equal(seq(x).features, bn(x.features))
    p = x.pad_to(9)                                        # row-wise: padding is allowed and carried
    y = seq(p)
    assert y.num_valid is p.num_valid and torch.equal(y.features[:6], bn(x.features))
    empty = spconv.SparseConvTensor(torch.zeros((0, 8)), torch.zeros((0, 4), dtype=torch.int32), [6, 6, 6], 1)
    assert seq(empty) is empty
    with pytest.raises(ValueError, match="features of shape"):
        MaskedBatchNorm1d(4).eval()(x)


def test_default_modules_still_refuse_and_plain_sparse_batchnorm_is_unchanged():
    p = _tensor(5).pad_to(8)
    with pytest.raises(NotImplementedError, match="padded SparseConvTensor"):
        spconv.SparseBatchNorm(8)(p)
    assert type(spconv.SparseBatchNorm(8).inner) is nn.BatchNorm1d
