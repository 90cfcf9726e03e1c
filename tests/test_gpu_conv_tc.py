"""wgmma conv engine (csrc/conv_tc.cu, conv_stem_tc.cu) through the C ABI (b200romp_conv2d, engine forced
to WGMMA) against a plain fp32 torch conv on the same bf16-rounded operands.  Covers every kernel family / epilogue:
1x1, 3x3 stride 1 (halo tile + shifted descriptors), 3x3 stride 2 (space-to-depth maps), direct epilogue (fp32 out,
fp32 residual, upsampled output, NCHW maps), bf16 out and bf16 residual,
multi-tile persistent loops, and the u8 stem.  Tolerance: fp32 accumulation of bf16 products - only the summation
order differs - plus one bf16 rounding of the output when it is stored as bf16 (2^-8 relative)."""
import numpy as np
import pytest
import torch

from romp_b200 import _lib
from romp_b200._lib import BF16, F32
from tests.gpu_util import conv2d, conv_ref

pytestmark = pytest.mark.gpu

# name, k, cin, cout, H, W, B, relu, res(0 none,1 f32,2 bf16), up, out_bf16, stride
CASES = [
    ("k1_c64_single", 1, 64, 64, 16, 8, 1, 0, 0, 1, 0, 1),
    ("k1_c64_multi", 1, 64, 64, 32, 32, 3, 1, 0, 1, 1, 1),
    ("k1_c256_n64", 1, 256, 64, 16, 16, 2, 0, 0, 1, 0, 1),
    ("k1_c128_n32_up4", 1, 128, 32, 16, 8, 2, 1, 1, 4, 1, 1),
    ("k1_c64_n256_res", 1, 64, 256, 16, 16, 2, 1, 2, 1, 1, 1),
    ("k3_c64_single", 3, 64, 64, 16, 8, 1, 0, 0, 1, 0, 1),
    ("k3_c64_multi_res", 3, 64, 64, 32, 24, 2, 1, 2, 1, 1, 1),
    ("k3_c32_res_many_tiles", 3, 32, 32, 64, 64, 40, 1, 2, 1, 1, 1),     # > 2 tiles per CTA and ring: double-buffered residual
    ("k3_c32", 3, 32, 32, 32, 16, 2, 1, 0, 1, 1, 1),
    # 32->32 on internal bf16 tensors runs pixel-pair folded (net.cu fold_pixel_pairs): borders, no relu, odd batch
    ("k3_c32_pairs_128", 3, 32, 32, 128, 128, 3, 1, 0, 1, 1, 1),
    ("k3_c32_pairs_norelu_res", 3, 32, 32, 16, 32, 3, 0, 2, 1, 1, 1),
    ("k3_c32_w48_unfolded", 3, 32, 32, 16, 48, 1, 1, 2, 1, 1, 1),        # odd tile count: stays on the unfolded kernels
    ("k3_c128_res", 3, 128, 128, 16, 16, 2, 1, 2, 1, 1, 1),
    ("k3_c256_res_many_tiles", 3, 256, 256, 16, 16, 24, 1, 2, 1, 1, 1),
    ("k3_c256_n32", 3, 256, 32, 32, 32, 1, 1, 0, 1, 1, 1),
    ("k3_c64_f32res_f32out", 3, 64, 64, 32, 16, 2, 1, 1, 1, 0, 1),
    ("s2_c64_single", 3, 64, 64, 32, 16, 1, 0, 0, 1, 0, 2),
    ("s2_c64_n128_res", 3, 64, 128, 64, 48, 2, 1, 2, 1, 1, 2),
    ("s2_c32_n32_f32res", 3, 32, 32, 64, 32, 2, 1, 1, 1, 1, 2),
    ("s2_c32_n192", 3, 32, 192, 32, 32, 2, 1, 0, 1, 1, 2),
    ("s2_c128_n256_res", 3, 128, 256, 32, 32, 2, 1, 2, 1, 1, 2),
    ("s2_c256_n64_many_tiles", 3, 256, 64, 64, 64, 20, 1, 0, 1, 1, 2),   # single-stage plan, one MMA warp
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_tcgen05_conv_matches_torch(case):
    name, k, cin, cout, H, W, B, relu, res_mode, up, out_bf16, stride = case
    rs = np.random.RandomState(len(name) * 131 + cin)
    x = torch.from_numpy(rs.normal(0, 1, (B, H, W, cin)).astype(np.float32)).cuda().bfloat16()
    w = torch.from_numpy(rs.normal(0, 1 / np.sqrt(cin * k * k), (cout, cin, k, k)).astype(np.float32)).bfloat16().float().numpy()
    b = rs.normal(0, 0.5, cout).astype(np.float32)
    res = None
    if res_mode:
        res = torch.from_numpy(rs.normal(0, 1, (B, H // stride * up, W // stride * up, cout)).astype(np.float32)).cuda()
        if res_mode == 2:
            res = res.bfloat16()
    got = conv2d(x, w, b, stride=stride, relu=bool(relu), res=res, up=up, out_dtype=BF16 if out_bf16 else F32,
                 engine=_lib.ENGINE_WGMMA).float().cpu()
    ref = conv_ref(x, w, b, stride=stride, relu=bool(relu), res=res, up=up)
    tol = 2e-4 + (2.0 ** -8) * ref.abs() if out_bf16 else 2e-4 + 1e-5 * ref.abs()
    bad = (got - ref).abs() > tol
    assert not bad.any(), f"{name}: {int(bad.sum())} of {bad.numel()} outputs off, max err {(got - ref).abs().max():.3e}"


def test_tcgen05_nchw_map_output_with_pow():
    """Head output convs write [B,C,H,W] fp32 maps with 1.1**x on the cam-scale channel (main.py:112-113)."""
    rs = np.random.RandomState(5)
    x = torch.from_numpy(rs.normal(0, 1, (2, 32, 32, 64)).astype(np.float32)).cuda().bfloat16()
    w = torch.from_numpy(rs.normal(0, 0.125, (35, 64, 1, 1)).astype(np.float32)).bfloat16().float().numpy()
    b = rs.normal(0, 0.5, 35).astype(np.float32)
    got = conv2d(x, w, b, out_dtype=F32, engine=_lib.ENGINE_WGMMA, out_nchw=1, pow_channel=0).cpu()
    ref = conv_ref(x, w, b, pow_channel=0).permute(0, 3, 1, 2)
    assert torch.allclose(got, ref, rtol=2e-5, atol=2e-4)


@pytest.mark.parametrize("B,H,W", [(1, 32, 16), (3, 64, 64), (5, 512, 512)])
def test_tcgen05_stem_u8(B, H, W):
    """backbone.conv1 on raw u8 frames, x/255*2-1 folded in (model.py:384-387); operand (x-127.5) is exact in bf16."""
    rs = np.random.RandomState(B)
    x = torch.from_numpy(rs.randint(0, 256, (B, H, W, 3)).astype(np.uint8)).cuda()
    w = rs.normal(0, 0.2, (64, 3, 3, 3)).astype(np.float32)
    b = rs.normal(0, 0.5, 64).astype(np.float32)
    got = conv2d(x, w, b, stride=2, relu=True, out_dtype=BF16, engine=_lib.ENGINE_WGMMA, input_norm=1).float().cpu()
    # the engine rounds w * 2/255 to bf16; use exactly those weights in the reference
    w_eff = (torch.from_numpy(w * (2.0 / 255.0)).bfloat16().float() * (255.0 / 2.0)).numpy()
    ref = conv_ref(x, w_eff, b, stride=2, relu=True, input_norm=1)
    tol = 3e-4 + (2.0 ** -8) * ref.abs()
    assert not ((got - ref).abs() > tol).any(), f"max err {(got - ref).abs().max():.3e}"


@pytest.mark.parametrize("cin,cout,B,out_bf16", [(2560, 512, 3, 1), (512, 512, 32, 1), (512, 128, 2, 0), (128, 128, 5, 1)])
def test_tcgen05_conv1d_streamed_weights(cin, cout, B, out_bf16):
    """BEV's bird's-eye Conv1d stack (bev/model.py:24-45,179-182) on the streamed-weight tensor-core engine (conv1d_tc.cu):
    [B,1,128,C] bf16, k = 3 along W, against torch conv on the same bf16-rounded operands."""
    rs = np.random.RandomState(cin + cout)
    x = torch.from_numpy(rs.normal(0, 1, (B, 1, 128, cin)).astype(np.float32)).cuda().bfloat16()
    w = torch.from_numpy(rs.normal(0, 1 / np.sqrt(cin * 3), (cout, cin, 3)).astype(np.float32)).bfloat16().float().numpy()
    b = rs.normal(0, 0.5, cout).astype(np.float32)
    got = conv2d(x, w, b, relu=True, out_dtype=BF16 if out_bf16 else F32, engine=_lib.ENGINE_WGMMA).float().cpu()
    ref = conv_ref(x, w, b, relu=True)
    tol = 3e-4 + (2.0 ** -8) * ref.abs() if out_bf16 else 3e-4 + 1e-5 * ref.abs()
    bad = (got - ref).abs() > tol
    assert not bad.any(), f"{int(bad.sum())} of {bad.numel()} outputs off, max err {(got - ref).abs().max():.3e}"


@pytest.mark.parametrize("k,cin,cout,hw", [(3, 32, 32, 32), (3, 64, 64, 32), (3, 128, 128, 16), (3, 256, 256, 16), (1, 64, 256, 32)])
def test_bf16_rounding_error_of_one_layer_is_bounded(k, cin, cout, hw):
    """What the bf16 engine costs per layer (the cases above compare on identical bf16-rounded operands and cannot see it):
    conv(bf16(x), bf16(w)) stored as bf16 against the fp32 conv of the UNROUNDED operands.  Each operand carries a relative
    rounding error <= 2^-9, the output one more: the relative L2 error of a layer must stay below 3 x 2^-9; a kernel that accumulated in bf16, or dropped K terms, would exceed it."""
    rs = np.random.RandomState(k * 1000 + cin)
    x = rs.normal(0, 1, (2, hw, hw, cin)).astype(np.float32)
    w = rs.normal(0, 1 / np.sqrt(cin * k * k), (cout, cin, k, k)).astype(np.float32)
    got = conv2d(torch.from_numpy(x).cuda().bfloat16(), w, None, out_dtype=BF16, engine=_lib.ENGINE_WGMMA).float().cpu()
    ref = conv_ref(torch.from_numpy(x), w)
    rel = float((got - ref).norm() / ref.norm())
    print(f"k{k} {cin}->{cout}: relative L2 error of the bf16 layer {rel:.2e}")
    assert rel < 3 * 2.0 ** -9
