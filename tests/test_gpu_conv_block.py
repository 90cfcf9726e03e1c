"""Fused HRNet BasicBlock (conv_block_tc.cu): relu(conv2(relu(conv1(x) + b1)) + b2 + x) as one op.

Each case builds the same block twice with NetBuilder: once as it is (the graph fuses it) and once with a second reader of
the intermediate tensor, which keeps the two convs apart on the per-conv wgmma path.  The fused block keeps the K order of
the per-conv kernel, so the two outputs must be bit-equal.  A comparison with the fp32 torch reference catches border bugs
both paths might share.  Frames of 64x128 make tiles touch every border; batch 5 makes the persistent CTAs loop over tiles,
batch 1 launches fewer tiles than SMs, and the folded block at batch 9 gives some CTAs a third tile."""
import numpy as np
import pytest
import torch

from romp_b200 import _lib
from romp_b200.graph import NetBuilder, round_bf16
from tests.gpu_util import conv_ref

pytestmark = pytest.mark.gpu

# name, C, batch, x channels, channel slice offset of the block (input and residual)
CASES = [
    ("c64", 64, 5, 64, 0),
    ("c32_pixel_pairs", 32, 5, 32, 0),
    ("c64_slice_64_of_192", 64, 5, 192, 64),
    ("c64_batch1", 64, 1, 64, 0),
    ("c32_pixel_pairs_batch1", 32, 1, 32, 0),
    ("c32_pixel_pairs_batch9", 32, 9, 32, 0),      # 288 folded tiles on 132 CTAs: a third tile (and parity wrap) per CTA
]
H, W = 64, 128


def _weights(C, seed):
    g = torch.Generator().manual_seed(seed)
    w1 = round_bf16((torch.randn(C, C, 3, 3, generator=g) / np.sqrt(9 * C)).numpy())
    w2 = round_bf16((torch.randn(C, C, 3, 3, generator=g) / np.sqrt(9 * C)).numpy())
    b1 = (0.1 * torch.randn(C, generator=g)).numpy()
    b2 = (0.1 * torch.randn(C, generator=g)).numpy()
    return w1, b1, w2, b2


def _run_block(C, B, xC, off, xin, weights, split):
    """-> (describe() op lines, block output [B, H, W, C] bf16)."""
    w1, b1, w2, b2 = weights
    nb = NetBuilder(0, "bf16")
    src = nb.tensor(H, W, xC, external=1)
    # the block's input must be an internal tensor (its TMA map is encoded at finalize): an exact identity 1x1 copy
    x = nb.conv(src, np.eye(xC, dtype=np.float32).reshape(xC, xC, 1, 1), None, engine=_lib.ENGINE_SIMT)
    t = nb.conv(x, w1, b1, relu=True, in_c_off=off)
    y = nb.conv(t, w2, b2, relu=True, res=x, res_c_off=off, name="y")
    if split:
        nb.maxpool(t)   # a second reader of the intermediate: the block stays two convs
    nb.finalize(B)
    _lib.check(nb.lib.b200romp_net_bind(nb.net, src, xin.data_ptr()), "bind")
    stream = torch.cuda.current_stream()
    _lib.check(nb.lib.b200romp_net_run(nb.net, B, stream.cuda_stream), "run")
    out = torch.empty(B, H, W, C, dtype=torch.bfloat16, device="cuda")
    _lib.check(nb.lib.b200romp_net_read_tensor(nb.net, y, B, out.data_ptr(), stream.cuda_stream), "read_tensor")
    torch.cuda.synchronize()
    lines = [l for l in nb.describe().splitlines() if l.startswith("op")]
    nb.lib.b200romp_net_destroy(nb.net)
    return lines, out.cpu()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fused_block_matches_per_conv_path(case):
    name, C, B, xC, off = case
    weights = _weights(C, 11)
    g = torch.Generator().manual_seed(3)
    xin = torch.randn(B, H, W, xC, generator=g).bfloat16().cuda()
    fused_ops, y_fused = _run_block(C, B, xC, off, xin, weights, split=False)
    split_ops, y_split = _run_block(C, B, xC, off, xin, weights, split=True)

    blocks = [l for l in fused_ops if " block " in l]
    assert len(blocks) == 1 and not [l for l in fused_ops if " k3 " in l and " block " not in l]
    assert not [l for l in split_ops if " block " in l] and len([l for l in split_ops if "wgmma   k3 s1" in l]) == 2
    if C == 32:   # both convs of the block run on pixel pairs, in either form
        assert blocks[0].count("pixel-pairs") == 2
        assert sum(l.count("pixel-pairs") for l in split_ops) == 2

    diff = (y_fused.float() - y_split.float()).abs().max().item()
    print(f"{name}: fused vs per-conv max|diff| {diff:.3e}")
    assert torch.equal(y_fused, y_split)

    w1, b1, w2, b2 = weights
    xs = xin.float().cpu()[..., off:off + C].contiguous()
    t_ref = conv_ref(xs, w1, b1, relu=True).bfloat16().float()
    ref = conv_ref(t_ref, w2, b2, relu=True, res=xs)
    tol = 2e-2 * float(ref.abs().max())
    err = (y_fused.float() - ref).abs().max().item()
    print(f"{name}: fused vs fp32 reference max|err| {err:.3e} (tol {tol:.1e})")
    assert err < tol
