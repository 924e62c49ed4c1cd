"""irsde_b200: H100-native (sm_90a) IR-SDE / Denoising-SDE reverse-diffusion sampler.

Public surface mirrors the reference (Algolzw/image-restoration-sde):
  * ``IRSDE`` / ``DenoisingSDE``            <- codes/utils/sde_utils.py
  * ``ConditionalUNet`` / ``DenoisingUNet``  <- codes/config/*/models/modules/DenoisingUNet_arch.py
  * ``ConditionalNAFNet`` / ``DenoisingNAFNet`` <- codes/config/*/models/modules/DenoisingNAFNet_arch.py
Importing the package does not need a GPU; running anything does (no CPU fallback).
"""
from . import _lib
from .sde import IRSDE, DenoisingSDE
from .unet import ConditionalUNet, DenoisingUNet, unet_param_shapes, infer_unet_config
from .nafnet import ConditionalNAFNet, DenoisingNAFNet, nafnet_param_shapes, infer_nafnet_config
from .shadow import adopt
from .latent import UNet, latent_unet_param_shapes
from . import imaging
from .imaging import tensor2img, calculate_psnr, calculate_ssim
from .pipeline import Restorer, plan_batches
from .refusion import TiledRefusion, tile_boxes, plan_units
from .dist import shard_range, sharded_reverse, broadcast_weights, NativeComm, comm_unique_id

__all__ = ["IRSDE", "DenoisingSDE", "ConditionalUNet", "DenoisingUNet", "ConditionalNAFNet", "DenoisingNAFNet", "UNet", "unet_param_shapes", "adopt", "infer_unet_config", "latent_unet_param_shapes",
           "nafnet_param_shapes", "infer_nafnet_config", "shard_range",
           "sharded_reverse", "broadcast_weights", "NativeComm", "comm_unique_id", "TiledRefusion", "tile_boxes", "plan_units", "imaging", "Restorer", "plan_batches", "tensor2img", "calculate_psnr", "calculate_ssim", "_lib"]
__version__ = "0.1"
