"""Fused ResNet Bottleneck (conv_bottleneck_tc.cu): relu(W3 relu(W2 * relu(W1 x + b1) + b2) + b3 + x) as one op.

Each case builds the same Bottleneck three times with NetBuilder: as it is (the graph fuses it); with a second reader of
each intermediate (still fused, and the kernel also writes both intermediates); and with conv2 on another concurrency lane,
which keeps the three convs apart on the per-conv wgmma path.  The fused kernel keeps the K order and the epilogue
arithmetic of the per-conv kernels, so the outputs, and the stored intermediates, must be bit-equal.  A comparison with the
fp32 torch reference catches border bugs all paths might share.  128 x 128 at batch 64 is HRNet's layer1 as the benchmark
runs it; batch 1 launches fewer tiles than SMs; 64 x 128 at batch 7 gives every CTA three or four tiles (and the x-stage
ring wraps at odd tile counts); 32 x 48 frames put most mid pixels of a tile outside the frame, where conv1's output must
be zero.
"""
import numpy as np
import pytest
import torch

from romp_b200 import _lib
from romp_b200.graph import NetBuilder, round_bf16
from tests.gpu_util import conv_ref

pytestmark = pytest.mark.gpu

# name, H, W, batch, x channels, channel slice offset of the block (input and residual)
CASES = [
    ("128x128_batch64", 128, 128, 64, 256, 0),
    ("64x128_batch1", 64, 128, 1, 256, 0),
    ("64x128_batch7", 64, 128, 7, 256, 0),   # 448 tiles on 132 CTAs
    ("32x48_batch3", 32, 48, 3, 256, 0),
    ("slice_256_of_320", 32, 48, 2, 320, 64),
]


def _weights(seed):
    g = torch.Generator().manual_seed(seed)
    w1 = round_bf16((torch.randn(64, 256, 1, 1, generator=g) / np.sqrt(256)).numpy())
    w2 = round_bf16((torch.randn(64, 64, 3, 3, generator=g) / np.sqrt(9 * 64)).numpy())
    w3 = round_bf16((torch.randn(256, 64, 1, 1, generator=g) / np.sqrt(64)).numpy())
    b1, b2, b3 = ((0.1 * torch.randn(c, generator=g)).numpy() for c in (64, 64, 256))
    return w1, b1, w2, b2, w3, b3


def _run_bottleneck(H, W, B, xC, off, xin, weights, mode):
    """mode "fused", "stored" (readers of t1 and t2 after the block) or "split" (conv2 on lane 1, and the same readers)
    -> (describe() op lines, launches, y [B, H, W, 256], t1 and t2 [B, H, W, 64] or None), all bf16 on the CPU"""
    w1, b1, w2, b2, w3, b3 = weights
    nb = NetBuilder(0, "bf16")
    src = nb.tensor(H, W, xC, external=1)
    # the block's input must be an internal tensor (its TMA map is encoded at finalize): an exact identity 1x1 copy
    x = nb.conv(src, np.eye(xC, dtype=np.float32).reshape(xC, xC, 1, 1), None, engine=_lib.ENGINE_SIMT)
    t1 = nb.conv(x, w1, b1, relu=True, in_c_off=off)
    with nb.on_lane(1 if mode == "split" else 0):
        t2 = nb.conv(t1, w2, b2, relu=True)
    y = nb.conv(t2, w3, b3, relu=True, res=x, res_c_off=off, name="y")
    if mode != "fused":
        nb.maxpool(t1)
        nb.maxpool(t2)
    nb.finalize(B)
    _lib.check(nb.lib.b200romp_net_bind(nb.net, src, xin.data_ptr()), "bind")
    stream = torch.cuda.current_stream()
    _lib.check(nb.lib.b200romp_net_run(nb.net, B, stream.cuda_stream), "run")

    def read(t, Cc):
        out = torch.empty(B, H, W, Cc, dtype=torch.bfloat16, device="cuda")
        _lib.check(nb.lib.b200romp_net_read_tensor(nb.net, t, B, out.data_ptr(), stream.cuda_stream), "read_tensor")
        return out

    outs = [read(y, 256)] + ([None, None] if mode == "fused" else [read(t1, 64), read(t2, 64)])
    torch.cuda.synchronize()
    lines = [l for l in nb.describe().splitlines() if l.startswith("op")]
    launches = nb.lib.b200romp_net_num_launches(nb.net)
    nb.lib.b200romp_net_destroy(nb.net)
    return (lines, launches) + tuple(None if o is None else o.cpu() for o in outs)


def x_id(conv_lines):
    """the block input's tensor id: conv3's residual"""
    return int(conv_lines[2].split(" res t")[1].split()[0])


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_bottleneck_matches_per_conv_path(case):
    name, H, W, B, xC, off = case
    weights = _weights(7)
    g = torch.Generator().manual_seed(4)
    xin = torch.randn(B, H, W, xC, generator=g).bfloat16().cuda()
    fused_ops, fused_n, y_fused, _, _ = _run_bottleneck(H, W, B, xC, off, xin, weights, "fused")
    stored_ops, stored_n, y_stored, t1_stored, t2_stored = _run_bottleneck(H, W, B, xC, off, xin, weights, "stored")
    split_ops, split_n, y_split, t1_split, t2_split = _run_bottleneck(H, W, B, xC, off, xin, weights, "split")

    # one launch, described as its three convs under one op number
    for ops, n in ((fused_ops, 2), (stored_ops, 4)):
        conv_lines = [l for l in ops if "[tc-bottleneck " in l]
        assert n == len(ops) - 2 and len(conv_lines) == 3 and len({l[:5] for l in conv_lines}) == 1, ops
        for k, (l, shape) in enumerate(zip(conv_lines, ("k1 s1  256->64 ", "k3 s1   64->64 ", "k1 s1   64->256 ")), 1):
            assert shape in l and f"[tc-bottleneck conv{k} of k1-k3-k1 grid " in l, l
        assert f"in t{x_id(conv_lines)}[" in conv_lines[0] and f"+{off} " in conv_lines[0]
    assert fused_n == 2 and stored_n == 4
    assert not [l for l in split_ops if "tc-bottleneck" in l] and split_n == 6
    for shape in ("wgmma   k1 s1  256->64 ", "wgmma   k3 s1   64->64 ", "wgmma   k1 s1   64->256 "):
        assert len([l for l in split_ops if shape in l]) == 1, split_ops

    assert torch.equal(t1_stored, t1_split) and torch.equal(t2_stored, t2_split)
    assert torch.equal(y_stored, y_split)
    diff = (y_fused.float() - y_split.float()).abs().max().item()
    print(f"{name}: fused vs per-conv max|diff| {diff:.3e}")
    assert torch.equal(y_fused, y_split)

    w1, b1, w2, b2, w3, b3 = weights
    frames = sorted({0, B - 1})
    xs = xin[frames].float().cpu()[..., off:off + 256].contiguous()
    t1 = conv_ref(xs, w1, b1, relu=True).bfloat16().float()
    t2 = conv_ref(t1, w2, b2, relu=True).bfloat16().float()
    ref = conv_ref(t2, w3, b3, relu=True, res=xs)
    tol = 2e-2 * float(ref.abs().max())
    err = (y_fused[frames].float() - ref).abs().max().item()
    print(f"{name}: fused vs fp32 reference max|err| {err:.3e} (tol {tol:.1e})")
    assert err < tol
