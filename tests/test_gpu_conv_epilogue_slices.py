"""NHWC epilogue of the wgmma conv engine (tc_device.cuh wg_epilogue_nhwc) on channel slices of wider tensors: the
output goes to channels [off, off + cout) of an out_C-channel tensor and the residual is read from the same slice of an
out_C-channel tensor, optionally broadcast from frame 0.  The channels outside the slice must be left untouched.  Covers the
bf16 residual (4 and 2 staged fragment rows at NT = 32 / 64) and the fp32 residual of the TF32 engine (2 / 1 rows)."""
import ctypes as C

import numpy as np
import pytest
import torch

from romp_b200 import _lib
from romp_b200._lib import BF16, F32, ConvDesc
from tests.gpu_util import TD, conv_ref, round_tf32

pytestmark = pytest.mark.gpu

# name, k, cin, cout, stride, out_C, off, dtype (bf16 = bf16 engine, f32 = TF32 engine), res_broadcast
CASES = [
    ("k1_bf16_n64_slice", 1, 64, 64, 1, 192, 64, BF16, 0),
    ("k3_bf16_n32_slice_bcast", 3, 32, 32, 1, 96, 32, BF16, 1),
    ("s2_bf16_n64_slice", 3, 64, 128, 2, 256, 128, BF16, 0),
    ("k1_tf32_n64_slice_bcast", 1, 64, 64, 1, 192, 64, F32, 1),
    ("k3_tf32_n32_slice", 3, 32, 32, 1, 96, 64, F32, 0),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_epilogue_writes_only_its_channel_slice(case):
    name, k, cin, cout, stride, out_C, off, dt, bcast = case
    B, H, W = 3, 32, 48
    g = torch.Generator().manual_seed(7)
    td = TD[dt]
    x = torch.randn(B, H, W, cin, generator=g).to(td).cuda()
    w = (torch.randn(cout, cin, k, k, generator=g) * (1.0 / np.sqrt(cin * k * k))).numpy()
    if dt == BF16:
        w = torch.from_numpy(w).to(torch.bfloat16).float().numpy()
    b = torch.randn(cout, generator=g).numpy()
    Ho, Wo = H // stride, W // stride
    res = torch.randn(B, Ho, Wo, out_C, generator=g).to(td).cuda()
    sentinel = 1024.0   # exact in bf16
    out = torch.full((B, Ho, Wo, out_C), sentinel, dtype=td, device="cuda")
    engine = _lib.ENGINE_WGMMA if dt == BF16 else _lib.ENGINE_TF32
    d = ConvDesc(0, 0, 0, off, -1, off, bcast, cin, cout, k, stride, 1, 1, 0, -1, engine)
    lib = _lib.load()
    rc = lib.b200romp_conv2d(C.byref(d), np.ascontiguousarray(w, np.float32).ctypes.data_as(C.POINTER(C.c_float)),
                             np.ascontiguousarray(b, np.float32).ctypes.data_as(C.POINTER(C.c_float)),
                             C.c_void_p(x.data_ptr()), dt, H, W, cin, C.c_void_p(out.data_ptr()), dt, out_C, 0,
                             C.c_void_p(res.data_ptr()), dt, B, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc, "conv2d")
    torch.cuda.synchronize()
    got = out.float().cpu()
    r = res.float().cpu()[:, :, :, off:off + cout]
    if bcast:
        r = r[:1].expand(B, -1, -1, -1)
    xr, wr = (x.float().cpu(), w) if dt == BF16 else (round_tf32(x.cpu()), round_tf32(torch.from_numpy(w)).numpy())
    ref = conv_ref(xr, wr, b, stride=stride, relu=True, res=r.contiguous())
    tol = 2e-2 * float(ref.abs().max()) if dt == BF16 else 1e-4 * float(ref.abs().max())
    err = (got[:, :, :, off:off + cout] - ref).abs().max().item()
    print(f"{name}: max|err| {err:.3e} (tol {tol:.1e})")
    assert err < tol
    assert (got[:, :, :, :off] == sentinel).all() and (got[:, :, :, off + cout:] == sentinel).all()
