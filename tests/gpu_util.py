import ctypes as C

import numpy as np
import torch

from romp_b200 import _lib
from romp_b200._lib import BF16, F32, U8, ConvDesc

TD = {F32: torch.float32, BF16: torch.bfloat16, U8: torch.uint8}


def conv2d(x_nhwc, w, b=None, *, stride=1, relu=False, res=None, up=1, out_dtype=F32, engine=_lib.ENGINE_SIMT,
           input_norm=0, out_nchw=0, pow_channel=-1, in_c_off=0, cin=None):
    """b200romp_conv2d on torch CUDA tensors; x [B,H,W,C] (f32/bf16/u8), w OIHW fp32 numpy."""
    lib = _lib.load()
    B, H, W, Cin_total = x_nhwc.shape
    if w.ndim == 3:                                   # Conv1d along W: [O, I, 3] -> ksize code 13 (1x3)
        cout, cin_w, _ = w.shape
        k, Ho, Wo = 13, H * up, W * up
    else:
        cout, cin_w, k, _ = w.shape
        Ho, Wo = ((H + 2 * (k // 2) - k) // stride + 1) * up, ((W + 2 * (k // 2) - k) // stride + 1) * up
    in_dt = {torch.float32: F32, torch.bfloat16: BF16, torch.uint8: U8}[x_nhwc.dtype]
    shape = (B, cout, Ho, Wo) if out_nchw else (B, Ho, Wo, cout)
    out = torch.empty(shape, dtype=TD[out_dtype], device=x_nhwc.device)
    d = ConvDesc(0, in_c_off, 0, 0, -1, 0, 0, cin_w, cout, k, stride, int(relu), up, input_norm, pow_channel, engine)
    wc = np.ascontiguousarray(w, dtype=np.float32)
    bc = None if b is None else np.ascontiguousarray(b, dtype=np.float32)
    res_dt = F32 if res is None else {torch.float32: F32, torch.bfloat16: BF16}[res.dtype]
    rc = lib.b200romp_conv2d(C.byref(d), wc.ctypes.data_as(C.POINTER(C.c_float)),
                             None if bc is None else bc.ctypes.data_as(C.POINTER(C.c_float)),
                             C.c_void_p(x_nhwc.data_ptr()), in_dt, H, W, Cin_total,
                             C.c_void_p(out.data_ptr()), out_dtype, cout, out_nchw,
                             None if res is None else C.c_void_p(res.data_ptr()), res_dt, B,
                             C.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc, "conv2d")
    torch.cuda.synchronize()
    return out


def conv_ref(x_nhwc, w, b=None, *, stride=1, relu=False, res=None, up=1, input_norm=0, pow_channel=-1, device="cpu",
             dtype=torch.float32):
    """torch reference of the fused op, computed in `dtype` on `device` (default: fp32 on the CPU); returns NHWC.
    w, b: numpy arrays or tensors; a residual with one frame is broadcast over the batch."""
    import torch.nn.functional as F
    x = x_nhwc.to(device=device, dtype=dtype).permute(0, 3, 1, 2)
    if input_norm:
        x = (x / 255.0) * 2.0 - 1.0
    wt = torch.as_tensor(w).to(device=device, dtype=dtype)
    bt = None if b is None else torch.as_tensor(b).to(device=device, dtype=dtype)
    if wt.ndim == 3:                                  # Conv1d along W
        y = F.conv2d(x, wt[:, :, None, :], bt, stride=1, padding=(0, 1))
    else:
        y = F.conv2d(x, wt, bt, stride=stride, padding=wt.shape[-1] // 2)
    if up > 1:
        y = F.interpolate(y, scale_factor=up, mode="nearest")
    if res is not None:
        y = y + res.to(device=device, dtype=dtype).permute(0, 3, 1, 2)
    if relu:
        y = F.relu(y)
    if pow_channel >= 0:
        y[:, pow_channel] = torch.pow(1.1, y[:, pow_channel])
    return y.permute(0, 2, 3, 1).contiguous()


def round_tf32(t):
    """fp32 -> TF32 (10 mantissa bits, ties away from zero) like cvt.rna.tf32.f32; stays in fp32 containers on t's device."""
    i = t.detach().float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)
