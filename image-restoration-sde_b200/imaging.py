"""Device-side versions of the image helpers the reference's test loops run on the CPU
(codes/utils/img_utils.py): ``tensor2img`` (:136-163), ``img2tensor`` (:171-180), ``calculate_psnr`` (:182-190),
``calculate_ssim`` (:217-234).  Same names, arguments and return types; the work runs in the native library
(uint8 quantisation / index maps / squared-error sums bit exact, SSIM fp64).  CPU inputs are staged to the
current CUDA device - there is no CPU implementation here."""
import ctypes
import math

import numpy as np
import torch

from . import _lib


def _bind():
    L = _lib.load()
    if getattr(L, "_img_bound", False):
        return L
    vp, i32, f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_double
    L.irsde_tensor2img_u8.argtypes = [vp, vp, i32, i32, i32, i32, f64, f64, vp]
    L.irsde_img2tensor_u8.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    L.irsde_sqerr_u8.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, vp]
    L.irsde_ssim_workspace.argtypes = [i32, i32, i32, i32, i32]
    L.irsde_ssim_workspace.restype = ctypes.c_int64
    L.irsde_ssim_u8.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, vp, vp]
    for f in (L.irsde_tensor2img_u8, L.irsde_img2tensor_u8, L.irsde_sqerr_u8, L.irsde_ssim_u8):
        f.restype = ctypes.c_int
    L._img_bound = True
    return L


def _cuda(t):
    if not torch.cuda.is_available():
        raise RuntimeError("irsde_b200.imaging runs on CUDA (sm_90a) only; there is no CPU path")
    return t if t.is_cuda else t.cuda(non_blocking=True)


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def tensor2img_device(tensor, min_max=(0, 1)):
    """fp32 [B,C,H,W] / [C,H,W] / [H,W] (RGB) -> uint8 CUDA tensor [B,H,W,C] / [H,W,C] / [H,W] (BGR)."""
    L = _bind()
    t = _cuda(tensor).float()
    shp = t.shape
    if t.dim() == 2:
        t4 = t[None, None]
    elif t.dim() == 3:
        t4 = t[None]
    elif t.dim() == 4:
        t4 = t
    else:
        raise TypeError("Only support 4D, 3D and 2D tensor. But received with dimension: {:d}".format(t.dim()))
    t4 = t4.contiguous()
    B, C, H, W = t4.shape
    out = torch.empty((B, H, W, C), dtype=torch.uint8, device=t4.device)
    with torch.cuda.device(t4.device):
        _lib.check(L.irsde_tensor2img_u8(ctypes.c_void_p(t4.data_ptr()), ctypes.c_void_p(out.data_ptr()), B, C, H, W,
                                         float(min_max[0]), float(min_max[1]), _stream(t4.device)))
    if len(shp) == 2:
        return out[0, :, :, 0]
    return out[0] if len(shp) == 3 else out


def tensor2img(tensor, out_type=np.uint8, min_max=(0, 1)):
    """Drop-in for ``util.tensor2img`` (single image; the reference's 4-D ``make_grid`` montage is not provided)."""
    if out_type != np.uint8:
        raise NotImplementedError("irsde_b200.tensor2img produces uint8 images")
    t = tensor.squeeze()
    if t.dim() == 4:
        raise NotImplementedError("batched tensors: use tensor2img_device (one image per batch entry)")
    return tensor2img_device(t, min_max).cpu().numpy()


def img2tensor_device(img):
    """uint8 [H,W,C] / [B,H,W,C] BGR (numpy or tensor) -> fp32 CUDA tensor [C,H,W] / [B,C,H,W] RGB in [0,1]."""
    L = _bind()
    a = torch.as_tensor(img)
    if a.dtype != torch.uint8:
        raise TypeError("img2tensor_device expects uint8 images")
    a = _cuda(a)
    single = a.dim() == 3
    a4 = (a[None] if single else a).contiguous()
    B, H, W, C = a4.shape
    out = torch.empty((B, C, H, W), dtype=torch.float32, device=a4.device)
    with torch.cuda.device(a4.device):
        _lib.check(L.irsde_img2tensor_u8(ctypes.c_void_p(a4.data_ptr()), ctypes.c_void_p(out.data_ptr()), B, C, H, W,
                                         _stream(a4.device)))
    return out[0] if single else out


def _pair_u8(img1, img2):
    a, b = torch.as_tensor(img1), torch.as_tensor(img2)
    for t in (a, b):
        if t.dtype != torch.uint8:
            raise TypeError("device metrics take uint8 images ([0,255]); quantise with tensor2img first")
    if a.shape != b.shape:
        raise ValueError("Input images must have the same dimensions.")
    a, b = _cuda(a), _cuda(b)
    if a.dim() == 2:
        a, b = a[None, :, :, None], b[None, :, :, None]
    elif a.dim() == 3:
        a, b = a[None], b[None]
    elif a.dim() != 4:
        raise ValueError("Wrong input image dimensions.")
    return a.contiguous(), b.contiguous()


def sqerr_device(img1, img2, crop_border=0):
    """Exact per-image sum of squared uint8 differences over the crop-bordered region: int64 CUDA tensor [B]."""
    L = _bind()
    a, b = _pair_u8(img1, img2)
    B, H, W, C = a.shape
    out = torch.empty((B,), dtype=torch.int64, device=a.device)
    with torch.cuda.device(a.device):
        _lib.check(L.irsde_sqerr_u8(ctypes.c_void_p(a.data_ptr()), ctypes.c_void_p(b.data_ptr()), B, H, W, C, int(crop_border),
                                    ctypes.c_void_p(out.data_ptr()), _stream(a.device)))
    return out


def calculate_psnr(img1, img2, crop_border=0):
    """Drop-in for ``util.calculate_psnr`` on uint8 images (numpy or tensors, one image): python float."""
    a, _ = _pair_u8(img1, img2)
    _, H, W, C = a.shape
    s = int(sqerr_device(img1, img2, crop_border)[0].item())
    n = (H - 2 * crop_border) * (W - 2 * crop_border) * C
    mse = np.float64(s) / n          # what np.mean of the float64 squares returns (all partial sums exact)
    if mse == 0:
        return float("inf")
    return 20 * math.log10(255.0 / math.sqrt(mse))


def ssim_device(img1, img2, crop_border=0):
    """Per-image mean SSIM (fp64 CUDA tensor [B]) of uint8 images."""
    L = _bind()
    a, b = _pair_u8(img1, img2)
    B, H, W, C = a.shape
    n = L.irsde_ssim_workspace(B, H, W, C, int(crop_border))
    if n <= 0:
        raise ValueError("SSIM needs at least 11x11 pixels after cropping")
    ws = torch.empty((n,), dtype=torch.float64, device=a.device)
    out = torch.empty((B,), dtype=torch.float64, device=a.device)
    with torch.cuda.device(a.device):
        _lib.check(L.irsde_ssim_u8(ctypes.c_void_p(a.data_ptr()), ctypes.c_void_p(b.data_ptr()), B, H, W, C, int(crop_border),
                                   ctypes.c_void_p(ws.data_ptr()), ctypes.c_void_p(out.data_ptr()), _stream(a.device)))
    return out


def calculate_ssim(img1, img2, crop_border=0):
    """Drop-in for ``util.calculate_ssim`` on uint8 images ([H,W], [H,W,1] or [H,W,3])."""
    return float(ssim_device(img1, img2, crop_border)[0].item())
