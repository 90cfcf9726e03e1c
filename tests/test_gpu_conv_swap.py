"""3x3 stride-1 bf16 convs with the weights as the wgmma A operand: 128 -> 128 with the slab resident (conv_tc.cu SWAP,
plan kind 31) and 256 -> 256 with the slab streamed beside the input (conv_tc_stream_kernel, plan kind 34).

Each case builds one conv net twice with NetBuilder: once with a bf16 output, which takes the weights-as-A plan, and once
with an fp32 output, which that plan does not cover, so that net runs the pixels-as-A plan.  Both plans keep the same K order
and apply bias, residual and ReLU to the same fp32 sums, so the bf16 output must equal the fp32 output rounded to bf16 bit
for bit.  The bf16 output is also checked against the float64 bound of test_gpu_graph_ops.  Frames of 32x32 at batch 8 give
every CTA one tile (64 tiles on the 66 CTAs of a 132-SM H100); 48x56 at batch 9 gives CTAs two or three tiles and tiles on
every border.  At 256 channels a work item is a 16x16 tile and one of the 4 slabs: 32x48 at batch 5 gives 120 items on 132
CTAs, at batch 9 216 items, one or two per CTA."""
import numpy as np
import pytest
import torch

from romp_b200 import _lib
from romp_b200._lib import BF16, F32
from romp_b200.graph import NetBuilder, round_bf16
from tests.test_gpu_graph_ops import conv_bound, excess

pytestmark = pytest.mark.gpu

SENTINEL = 1024.0   # exact in bf16: the channels outside an output slice must keep it
# name, conv channels, batch, H, W, x channels (input slice at x_off), residual: None or (channels, offset, dtype,
# broadcast), out channels, out offset
CASES = [
    ("b64_32x32", 128, 64, 32, 32, 128, 0, None, 128, 0),
    ("b64_32x32_res", 128, 64, 32, 32, 128, 0, (128, 0, BF16, 0), 128, 0),
    ("b1_32x32_res", 128, 1, 32, 32, 128, 0, (128, 0, BF16, 0), 128, 0),
    ("b8_one_tile_per_cta", 128, 8, 32, 32, 128, 0, (128, 0, BF16, 0), 128, 0),
    ("b9_48x56_uneven_tiles", 128, 9, 48, 56, 128, 0, (128, 0, BF16, 0), 128, 0),
    ("slices_bf16_res", 128, 5, 32, 48, 256, 64, (192, 64, BF16, 0), 384, 128),
    ("slices_f32_res_bcast", 128, 5, 32, 48, 256, 128, (256, 32, F32, 1), 256, 64),
    ("c256_b64_16x16", 256, 64, 16, 16, 256, 0, None, 256, 0),
    ("c256_b64_16x16_res", 256, 64, 16, 16, 256, 0, (256, 0, BF16, 0), 256, 0),
    ("c256_b1_16x16_res", 256, 1, 16, 16, 256, 0, (256, 0, BF16, 0), 256, 0),
    ("c256_b5_32x48_one_item_per_cta", 256, 5, 32, 48, 256, 0, (256, 0, BF16, 0), 256, 0),
    ("c256_b9_32x48_uneven_items", 256, 9, 32, 48, 256, 0, (256, 0, BF16, 0), 256, 0),
    ("c256_slices_f32_res_bcast", 256, 5, 32, 48, 320, 64, (384, 64, F32, 1), 384, 128),
]
# the weights-as-A plan and the pixels-as-A plan each conv width takes, as describe() names them
PLANS = {128: ("[tc k3 v1 nt64", "[tc-swap", "[tc k3 v0 nt64"), 256: ("[tc k3 v4 nt64", "[tc-stream", "[tc k3 v0 nt32")}
TD = {BF16: torch.bfloat16, F32: torch.float32}


def _run(case, x, res, w, b, out_dtype):
    """-> (describe() line of the 3x3 conv, the whole output tensor on the CPU)"""
    name, C, B, H, W, xC, x_off, rs, oC, o_off = case
    nb = NetBuilder(0, "bf16")
    src = nb.tensor(H, W, xC, external=1)
    # the conv's input must be an internal tensor (its TMA map is encoded at finalize): an exact identity 1x1 copy
    xi = nb.conv(src, np.eye(xC, dtype=np.float32).reshape(xC, xC, 1, 1), None, engine=_lib.ENGINE_SIMT)
    out_t = nb.tensor(H, W, oC, out_dtype, external=1)
    kw = {}
    if rs is not None:
        rC, r_off, r_dt, bcast = rs
        kw = dict(res=nb.tensor(H, W, rC, r_dt, external=1), res_c_off=r_off, res_broadcast=bcast)
    nb.conv(xi, w, b, relu=True, in_c_off=x_off, out=out_t, out_c_off=o_off, **kw)
    nb.finalize(B)
    out = torch.full((B, H, W, oC), SENTINEL, dtype=TD[out_dtype], device="cuda")
    _lib.check(nb.lib.b200romp_net_bind(nb.net, src, x.data_ptr()), "bind")
    _lib.check(nb.lib.b200romp_net_bind(nb.net, out_t, out.data_ptr()), "bind")
    if rs is not None:
        _lib.check(nb.lib.b200romp_net_bind(nb.net, kw["res"], res.data_ptr()), "bind")
    _lib.check(nb.lib.b200romp_net_run(nb.net, B, torch.cuda.current_stream().cuda_stream), "run")
    torch.cuda.synchronize()
    lines = [l for l in nb.describe().splitlines() if l.startswith("op") and " k3 " in l]
    nb.lib.b200romp_net_destroy(nb.net)
    assert len(lines) == 1
    return lines[0], out.cpu()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_swapped_plan_matches_pixels_as_a_plan(case):
    name, C, B, H, W, xC, x_off, rs, oC, o_off = case
    g = torch.Generator().manual_seed(5)
    w = round_bf16((torch.randn(C, C, 3, 3, generator=g) / np.sqrt(9 * C)).numpy())
    b = (0.1 * torch.randn(C, generator=g)).numpy()
    x = torch.randn(B, H, W, xC, generator=g).bfloat16().cuda()
    res = None
    if rs is not None:
        rC, r_off, r_dt, bcast = rs
        res = torch.randn(1 if bcast else B, H, W, rC, generator=g).to(TD[r_dt]).cuda()

    line_new, y_new = _run(case, x, res, w, b, BF16)
    line_old, y_old = _run(case, x, res, w, b, F32)
    new_plan, new_tag, old_plan = PLANS[C]
    assert new_plan in line_new and new_tag in line_new, line_new
    assert old_plan in line_old and new_tag not in line_old, line_old

    sl = slice(o_off, o_off + C)
    assert torch.equal(y_new[..., :o_off], torch.full_like(y_new[..., :o_off], SENTINEL))
    assert torch.equal(y_new[..., o_off + C:], torch.full_like(y_new[..., o_off + C:], SENTINEL))
    diff = (y_new[..., sl].float() - y_old[..., sl]).abs().max().item()
    print(f"{name}: swapped vs pixels-as-A max|diff| {diff:.3e}")
    assert torch.equal(y_new[..., sl], y_old[..., sl].bfloat16())

    x64 = x[..., x_off:x_off + C].double()
    r64 = None if rs is None else res[..., rs[1]:rs[1] + C].double()
    v, bound = conv_bound(x64, torch.from_numpy(w).double().cuda(), torch.from_numpy(b).double().cuda(), relu=True, res=r64,
                          out_dt=BF16)
    worst, over = excess(y_new[..., sl].cuda(), v, bound)
    print(f"{name}: worst |err| / fp64 bound {worst:.3f}")
    assert over == 0
