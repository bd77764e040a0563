"""VGG11-BN feature pyramid on the sm_90a kernels (reference: network/pretrain_models.py:17-31
VGGBNPretrain and :61-72 VGGBNPretrainV3; layer table :86-111).

Eval-mode BatchNorm is folded into the packed conv weights/bias at pack time
(w' = w * gamma/sqrt(var+eps), b' = (b - mean) * gamma/sqrt(var+eps) + beta); ReLU is the conv
epilogue, except after the last conv of the 1/16 block which the reference leaves pre-ReLU
(features[21:27] stops before index 27).
"""
import torch

from .. import ops
from .params import VGG11_BLOCKS

BN_EPS = 1e-5


def pack_vgg(params):
    """params: VGG11BNParams on the GPU.  Returns {conv_slot: PackedConv} with BN folded in."""
    packed = {}
    f = params.features
    with torch.no_grad():
        for block in VGG11_BLOCKS:
            for slot in block:
                conv, bn = f[slot], f[slot + 1]
                scale = (bn.weight / torch.sqrt(bn.running_var + BN_EPS)).float().contiguous()
                bias = ((conv.bias - bn.running_mean) * scale + bn.bias).float().contiguous()
                packed[slot] = ops.pack_conv(conv.weight, stride=1, pad=1, cout_scale=scale, bias_override=bias)
    return packed


def vgg_pyramid(packed, x, full_res=False):
    """x: [N, H, W, 4] ImageNet-normalised, channel 3 zero.  Returns the six maps
    [1/1 (None unless full_res), 1/2, 1/4, 1/8, 1/16 (pre-ReLU), 1/32 (max-pool of the pre-ReLU map)],
    channels-last.  Nothing on the inference path reads the 1/1 map, so the first conv, its ReLU and the
    first max-pool run as one kernel (g6d_vgg_first_block) that never writes it."""
    outs = []
    fused = not full_res and x.shape[1] % 2 == 0 and x.shape[2] % 2 == 0 and x.shape[3] == 4
    for bi, block in enumerate(VGG11_BLOCKS):
        if bi == 0 and fused:
            outs.append(None)
            x = ops.vgg_first_block(x, packed[block[0]])
            continue
        if bi > 0 and not (bi == 1 and fused):
            x = ops.maxpool2x2(x)
        for slot in block:
            # reuse_im2col: the small maps the A-reuse kernel would take run on the persistent kernel with TMA
            # im2col A instead, in its K order (bit-identical); the larger maps are planned as without it
            x = ops.conv(x, packed[slot], act=ops.ACT_NONE if slot == 25 else ops.ACT_RELU, reuse_im2col=True,
                         fold_splits=True)
        outs.append(x)
    outs.append(ops.maxpool2x2(x))
    return outs


def vgg_v1(packed, x):
    """(1/8, 1/16 pre-ReLU, 1/32): what the detector and selector consume."""
    p = vgg_pyramid(packed, x)
    return p[3], p[4], p[5]


def vgg_v3(packed, x):
    """(1/4, 1/8, 1/16 pre-ReLU): what the refiner consumes."""
    p = vgg_pyramid(packed, x)
    return p[2], p[3], p[4]
