"""The 32-channel fused BasicBlock (conv_block_tc.cu, pixel-pair folded, with the compact weight image that keeps only
the tap halves its MMAs read) across frame sizes and batches whose tile count is not a multiple of the grid.

The persistent CTAs loop over tiles with one input stage and one mid buffer whose barrier parities flip per tile, so odd
batches and frame sizes with 3 x 3 or 2 x 5 tiles per frame give CTAs of 1, 2, 3, 4 and 5 tiles in one launch.  Every
output must equal the unfused two-conv net bit for bit and lie within the float64 bound of the graph checks
(test_gpu_graph_ops.block_bound)."""
import numpy as np
import pytest
import torch

from romp_b200 import _lib
from romp_b200.graph import NetBuilder, round_bf16
from tests.test_gpu_graph_ops import block_bound, excess

pytestmark = pytest.mark.gpu

C = 32
# frame H x W, batch: the folded block's 16 x 16 tiles of pixel pairs cover 16 x 32 pixels, (W / 32) * (H / 16) per frame
CASES = [
    (64, 128, 3),     # 48 tiles: fewer than SMs, every CTA runs one tile
    (48, 96, 17),     # 153 tiles of 3 x 3 per frame: one or two per CTA
    (48, 96, 31),     # 279 tiles: two or three per CTA
    (80, 64, 29),     # 290 tiles of 2 x 5 per frame: two or three per CTA
    (64, 128, 41),    # 656 tiles: four or five per CTA
]


def _weights(seed):
    g = torch.Generator().manual_seed(seed)
    w1 = round_bf16((torch.randn(C, C, 3, 3, generator=g) / np.sqrt(9 * C)).numpy())
    w2 = round_bf16((torch.randn(C, C, 3, 3, generator=g) / np.sqrt(9 * C)).numpy())
    b1 = (0.1 * torch.randn(C, generator=g)).numpy()
    b2 = (0.1 * torch.randn(C, generator=g)).numpy()
    return w1, b1, w2, b2


def _run_block(H, W, B, xin, weights, split):
    """-> (describe() op lines, block output [B, H, W, C] bf16).  split adds a second reader of the intermediate, which
    keeps the two convs apart on the per-conv path."""
    w1, b1, w2, b2 = weights
    nb = NetBuilder(0, "bf16")
    src = nb.tensor(H, W, C, external=1)
    # the block's input must be an internal tensor (its TMA map is encoded at finalize): an exact identity 1x1 copy
    x = nb.conv(src, np.eye(C, dtype=np.float32).reshape(C, C, 1, 1), None, engine=_lib.ENGINE_SIMT)
    t = nb.conv(x, w1, b1, relu=True)
    y = nb.conv(t, w2, b2, relu=True, res=x, name="y")
    if split:
        nb.maxpool(t)
    nb.finalize(B)
    _lib.check(nb.lib.b200romp_net_bind(nb.net, src, xin.data_ptr()), "bind")
    stream = torch.cuda.current_stream()
    _lib.check(nb.lib.b200romp_net_run(nb.net, B, stream.cuda_stream), "run")
    out = torch.empty(B, H, W, C, dtype=torch.bfloat16, device="cuda")
    _lib.check(nb.lib.b200romp_net_read_tensor(nb.net, y, B, out.data_ptr(), stream.cuda_stream), "read_tensor")
    torch.cuda.synchronize()
    lines = [l for l in nb.describe().splitlines() if l.startswith("op")]
    nb.lib.b200romp_net_destroy(nb.net)
    return lines, out


@pytest.mark.parametrize("H,W,B", CASES, ids=[f"{h}x{w}_b{b}" for h, w, b in CASES])
def test_folded_block_tile_counts(H, W, B):
    weights = _weights(H * 1000 + B)
    g = torch.Generator().manual_seed(B)
    xin = torch.randn(B, H, W, C, generator=g).bfloat16().cuda()
    fused_ops, y_fused = _run_block(H, W, B, xin, weights, split=False)
    split_ops, y_split = _run_block(H, W, B, xin, weights, split=True)

    blocks = [l for l in fused_ops if " block " in l]
    assert len(blocks) == 1 and blocks[0].count("pixel-pairs") == 2
    assert not [l for l in split_ops if " block " in l]
    tiles = (W // 32) * (H // 16) * B
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"{H}x{W} batch {B}: {tiles} tiles on {min(tiles, sms)} CTAs, {-(-tiles // sms)} on CTA 0")

    assert torch.equal(y_fused, y_split), f"fused vs per-conv max|diff| {(y_fused.float() - y_split.float()).abs().max().item():.3e}"

    w1, b1, w2, b2 = (torch.from_numpy(np.asarray(a, dtype=np.float32)).cuda().double() for a in weights)
    v, bound = block_bound(xin.double(), w1, b1, w2, b2)
    worst, over = excess(y_fused, v, bound)
    print(f"{H}x{W} batch {B}: worst |err|/bound {worst:.3f}")
    assert over == 0
