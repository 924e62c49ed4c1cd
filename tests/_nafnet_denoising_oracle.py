"""CPU oracle of the denoising-sde task's ConditionalNAFNet (tests/ is on sys.path under pytest's default import mode).

That network differs from the deraining one only before the first block: its intro conv reads x's img_channel channels
instead of cat(x - cond, cond), and forward(x, time) takes no condition
(codes/config/denoising-sde/models/modules/DenoisingNAFNet_arch.py:103,147-150).  Everything from intro on is
restated with the shared oracle's NAFBlock (oracle/irsde_oracle.py: naf_block, DenoisingNAFNet_arch.py:51-84).
"""
import math

import torch
import torch.nn.functional as F

from oracle import irsde_oracle as O


def forward(P, x, time, width, enc_blk_nums, middle_blk_num, dec_blk_nums):
    """ConditionalNAFNet.forward of the denoising-sde task: DenoisingNAFNet_arch.py:147-184 (zero pad, crop)."""
    if isinstance(time, (int, float)):
        time = torch.tensor([time])
    time = time.reshape(-1)
    half = width // 2
    freqs = torch.exp(torch.arange(half) * -(math.log(10000) / (half - 1)))
    emb = time[:, None] * freqs[None, :]
    emb = torch.cat((emb.sin(), emb.cos()), dim=-1)
    t = F.linear(emb, P["time_mlp.1.weight"], P["time_mlp.1.bias"])
    t = F.linear(O._gate(t, dim=-1), P["time_mlp.3.weight"], P["time_mlp.3.bias"])
    H, W = x.shape[2:]
    s = 2 ** len(enc_blk_nums)
    x = F.pad(x, (0, (s - W % s) % s, 0, (s - H % s) % s))  # zero pad (not reflect)
    x = F.conv2d(x, P["intro.weight"], P["intro.bias"], padding=1)
    encs = []
    for i, num in enumerate(enc_blk_nums):
        for j in range(num):
            x = O.naf_block(P, "encoders.%d.%d." % (i, j), x, t)
        encs.append(x)
        x = F.conv2d(x, P["downs.%d.weight" % i], P["downs.%d.bias" % i], stride=2)
    for j in range(middle_blk_num):
        x = O.naf_block(P, "middle_blks.%d." % j, x, t)
    for i, num in enumerate(dec_blk_nums):
        x = F.pixel_shuffle(F.conv2d(x, P["ups.%d.0.weight" % i]), 2)
        x = x + encs[len(encs) - 1 - i]
        for j in range(num):
            x = O.naf_block(P, "decoders.%d.%d." % (i, j), x, t)
    x = F.conv2d(x, P["ending.weight"], P["ending.bias"], padding=1)
    return x[..., :H, :W]


def param_shapes(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums):
    """The conditional layout with intro.weight reading img_channel channels (DenoisingNAFNet_arch.py:103)."""
    S = O.nafnet_param_shapes(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums)
    S["intro.weight"] = (width, img_channel, 3, 3)
    return S


def make_weights(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums, seed=0):
    """The shared oracle's random NAFNet weights (nonzero beta / gamma), with an intro conv of this layout."""
    P = O.make_nafnet_weights(img_channel, width, middle_blk_num, enc_blk_nums, dec_blk_nums, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    fan_in = img_channel * 9
    P["intro.weight"] = (torch.rand(width, img_channel, 3, 3, generator=g) * 2 - 1) * math.sqrt(3.0 / fan_in)
    return P
