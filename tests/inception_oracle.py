"""Functional restatement of the scoring networks INCEPTION_V3.forward and INCEPTION_V3_FID.forward (ref:
image_generation/model.py:290-451) and of get_activations' pooling (utils.py:587-641) over a state_dict with
torchvision's Inception3 keys, in torch (any device, fp32 / fp64) with torch.nn.functional only.  The trunk functions
are oracle/image_encoder_oracle.py's.  Python constants enter each op as the reference writes them, so in fp32 the
rounding follows the reference's tensor ops."""
import torch
import torch.nn.functional as F

from oracle import image_encoder_oracle as E

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
FID_DIMS = {64: 0, 192: 1, 768: 2, 2048: 3}


def _tv(sd):
    """torchvision keys: INCEPTION_V3's ``model.`` prefix dropped."""
    return {(k[len("model."):] if k.startswith("model.") else k): v for k, v in sd.items()}


def _stem(sd, x, upto):
    """Conv2d_1a_3x3 .. the first (upto 0) or second (upto 1) max-pool."""
    x = E.basic_conv(sd, "Conv2d_1a_3x3", x, stride=2)
    x = E.basic_conv(sd, "Conv2d_2a_3x3", x)
    x = E.basic_conv(sd, "Conv2d_2b_3x3", x, padding=1)
    x = F.max_pool2d(x, kernel_size=3, stride=2)
    outs = [x]
    if upto >= 1:
        x = E.basic_conv(sd, "Conv2d_3b_1x1", x)
        x = E.basic_conv(sd, "Conv2d_4a_3x3", x)
        x = F.max_pool2d(x, kernel_size=3, stride=2)
        outs.append(x)
    return outs


def inception_v3_forward(sd, x):
    """ref: model.py:301-315 (torchvision Inception3 in eval mode, transform_input=False).  x (B, 3, H, W) in [-1, 1]
    -> (B, 1000) probabilities in x's dtype."""
    sd = _tv(sd)
    x = x * 0.5 + 0.5
    x = torch.stack([(x[:, c] - MEAN[c]) / STD[c] for c in range(3)], 1)
    x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=True)
    x = _stem(sd, x, 1)[-1]
    for name, blk in E.BLOCKS:
        x = blk(sd, name, x)
    x = F.adaptive_avg_pool2d(x, (1, 1)).flatten(1)          # dropout: identity in eval
    x = F.linear(x, sd["fc.weight"].to(x.dtype), sd["fc.bias"].to(x.dtype))
    return F.softmax(x, dim=-1)


def inception_fid_forward(sd, x, blocks):
    """ref: model.py:416-451.  x (B, 3, H, W) in [-1, 1] -> the maps of the requested blocks (sorted), block 3 as
    (B, 2048, 1, 1)."""
    sd = _tv(sd)
    blocks = sorted(blocks)
    last = blocks[-1]
    x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False)
    x = x * 0.5 + 0.5
    x = torch.stack([x[:, c] * (STD[c] / 0.5) + (MEAN[c] - 0.5) / 0.5 for c in range(3)], 1)
    maps = _stem(sd, x, min(last, 1))
    if last >= 2:
        x = maps[-1]
        for name, blk in E.BLOCKS[:8]:
            x = blk(sd, name, x)
        maps.append(x)
    if last >= 3:
        for name, blk in E.BLOCKS[8:]:
            x = blk(sd, name, x)
        maps.append(F.adaptive_avg_pool2d(x, (1, 1)))
    return [maps[b] for b in blocks]


def fid_activations(sd, x, dims):
    """get_activations of one batch: the block's map averaged over its pixels, (B, dims)."""
    m = inception_fid_forward(sd, x, [FID_DIMS[dims]])[0]
    return F.adaptive_avg_pool2d(m, (1, 1)).flatten(1)


def inception3_test_state_dict(keys_shapes, seed=0):
    """Weights for the tests over torchvision's Inception3 keys: the trunk as oracle.test_state_dict draws it, ``fc``
    scaled so that the logits spread by O(1) (the default initialisation saturates the softmax: a probability of 1.0
    makes the Inception score nan), the auxiliary head's ``fc`` likewise."""
    trunk = {k: v for k, v in keys_shapes.items() if not k.endswith(("fc.weight", "fc.bias"))}
    out = E.test_state_dict(trunk, seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k, v in keys_shapes.items():
        if k.endswith("fc.weight"):
            out[k] = torch.randn(v.shape, generator=g) * (4.0 / v.shape[1]) ** 0.5
        elif k.endswith("fc.bias"):
            out[k] = 0.1 * torch.randn(v.shape, generator=g)
    return {k: out[k] for k in keys_shapes}
