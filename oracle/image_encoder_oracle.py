"""Functional restatement of the DAMSM image encoder CNN_ENCODER.forward (ref: image_generation/model.py:182-287) over
a state_dict, in torch-CPU (or any device) fp32 / fp64 with torch.nn.functional only, so it runs without torchvision.
The trunk is torchvision's Inception-v3 (torchvision/models/inception.py: BasicConv2d, InceptionA-E) from
Conv2d_1a_3x3 to Mixed_7c, with every BatchNorm in eval mode (the reference freezes the encoder and calls eval():
trainer.py:75-89, evaluator.py:97-105)."""
import torch
import torch.nn.functional as F

BN_EPS = 0.001      # torchvision BasicConv2d: nn.BatchNorm2d(out_channels, eps=0.001)


def basic_conv(sd, p, x, stride=1, padding=0, stats=None):
    """torchvision BasicConv2d.forward: relu(bn(conv(x))), conv without bias, bn in eval mode."""
    w = sd[p + ".conv.weight"].to(x.dtype)
    y = F.conv2d(x, w, None, stride, padding)
    y = F.batch_norm(y, sd[p + ".bn.running_mean"].to(x.dtype), sd[p + ".bn.running_var"].to(x.dtype),
                     sd[p + ".bn.weight"].to(x.dtype), sd[p + ".bn.bias"].to(x.dtype), False, 0.0, BN_EPS)
    y = F.relu(y)
    if stats is not None:
        stats.append((p, y.detach().abs().max().item()))
    return y


def inception_a(sd, p, x, st=None):
    b1 = basic_conv(sd, p + ".branch1x1", x, stats=st)
    b5 = basic_conv(sd, p + ".branch5x5_2", basic_conv(sd, p + ".branch5x5_1", x, stats=st), padding=2, stats=st)
    b3 = basic_conv(sd, p + ".branch3x3dbl_1", x, stats=st)
    b3 = basic_conv(sd, p + ".branch3x3dbl_2", b3, padding=1, stats=st)
    b3 = basic_conv(sd, p + ".branch3x3dbl_3", b3, padding=1, stats=st)
    bp = basic_conv(sd, p + ".branch_pool", F.avg_pool2d(x, 3, 1, 1), stats=st)
    return torch.cat([b1, b5, b3, bp], 1)


def inception_b(sd, p, x, st=None):
    b3 = basic_conv(sd, p + ".branch3x3", x, stride=2, stats=st)
    bd = basic_conv(sd, p + ".branch3x3dbl_1", x, stats=st)
    bd = basic_conv(sd, p + ".branch3x3dbl_2", bd, padding=1, stats=st)
    bd = basic_conv(sd, p + ".branch3x3dbl_3", bd, stride=2, stats=st)
    return torch.cat([b3, bd, F.max_pool2d(x, 3, 2)], 1)


def inception_c(sd, p, x, st=None):
    b1 = basic_conv(sd, p + ".branch1x1", x, stats=st)
    b7 = basic_conv(sd, p + ".branch7x7_1", x, stats=st)
    b7 = basic_conv(sd, p + ".branch7x7_2", b7, padding=(0, 3), stats=st)
    b7 = basic_conv(sd, p + ".branch7x7_3", b7, padding=(3, 0), stats=st)
    bd = basic_conv(sd, p + ".branch7x7dbl_1", x, stats=st)
    bd = basic_conv(sd, p + ".branch7x7dbl_2", bd, padding=(3, 0), stats=st)
    bd = basic_conv(sd, p + ".branch7x7dbl_3", bd, padding=(0, 3), stats=st)
    bd = basic_conv(sd, p + ".branch7x7dbl_4", bd, padding=(3, 0), stats=st)
    bd = basic_conv(sd, p + ".branch7x7dbl_5", bd, padding=(0, 3), stats=st)
    bp = basic_conv(sd, p + ".branch_pool", F.avg_pool2d(x, 3, 1, 1), stats=st)
    return torch.cat([b1, b7, bd, bp], 1)


def inception_d(sd, p, x, st=None):
    b3 = basic_conv(sd, p + ".branch3x3_2", basic_conv(sd, p + ".branch3x3_1", x, stats=st), stride=2, stats=st)
    b7 = basic_conv(sd, p + ".branch7x7x3_1", x, stats=st)
    b7 = basic_conv(sd, p + ".branch7x7x3_2", b7, padding=(0, 3), stats=st)
    b7 = basic_conv(sd, p + ".branch7x7x3_3", b7, padding=(3, 0), stats=st)
    b7 = basic_conv(sd, p + ".branch7x7x3_4", b7, stride=2, stats=st)
    return torch.cat([b3, b7, F.max_pool2d(x, 3, 2)], 1)


def inception_e(sd, p, x, st=None):
    b1 = basic_conv(sd, p + ".branch1x1", x, stats=st)
    b3 = basic_conv(sd, p + ".branch3x3_1", x, stats=st)
    b3 = torch.cat([basic_conv(sd, p + ".branch3x3_2a", b3, padding=(0, 1), stats=st),
                    basic_conv(sd, p + ".branch3x3_2b", b3, padding=(1, 0), stats=st)], 1)
    bd = basic_conv(sd, p + ".branch3x3dbl_1", x, stats=st)
    bd = basic_conv(sd, p + ".branch3x3dbl_2", bd, padding=1, stats=st)
    bd = torch.cat([basic_conv(sd, p + ".branch3x3dbl_3a", bd, padding=(0, 1), stats=st),
                    basic_conv(sd, p + ".branch3x3dbl_3b", bd, padding=(1, 0), stats=st)], 1)
    bp = basic_conv(sd, p + ".branch_pool", F.avg_pool2d(x, 3, 1, 1), stats=st)
    return torch.cat([b1, b3, bd, bp], 1)


BLOCKS = [("Mixed_5b", inception_a), ("Mixed_5c", inception_a), ("Mixed_5d", inception_a), ("Mixed_6a", inception_b),
          ("Mixed_6b", inception_c), ("Mixed_6c", inception_c), ("Mixed_6d", inception_c), ("Mixed_6e", inception_c),
          ("Mixed_7a", inception_d), ("Mixed_7b", inception_e), ("Mixed_7c", inception_e)]


def cnn_encoder_forward(sd, x, stats=None):
    """ref: model.py:227-287.  x (B, 3, H, W) -> (features (B, nef, 17, 17), cnn_code (B, nef)) in x's dtype.
    ``stats``: optional list that receives (layer, max|activation|) of every BasicConv2d."""
    x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=True)      # model.py:230
    x = basic_conv(sd, "Conv2d_1a_3x3", x, stride=2, stats=stats)                     # model.py:232
    x = basic_conv(sd, "Conv2d_2a_3x3", x, stats=stats)                               # model.py:234
    x = basic_conv(sd, "Conv2d_2b_3x3", x, padding=1, stats=stats)                    # model.py:236
    x = F.max_pool2d(x, kernel_size=3, stride=2)                                       # model.py:238
    x = basic_conv(sd, "Conv2d_3b_1x1", x, stats=stats)                               # model.py:240
    x = basic_conv(sd, "Conv2d_4a_3x3", x, stats=stats)                               # model.py:242
    x = F.max_pool2d(x, kernel_size=3, stride=2)                                       # model.py:245
    features = None
    for name, blk in BLOCKS:                                                           # model.py:248-273
        x = blk(sd, name, x, stats)
        if name == "Mixed_6e":
            features = x                                                               # model.py:266
    x = F.avg_pool2d(x, kernel_size=8).view(x.size(0), -1)                            # model.py:275-279
    cnn_code = F.linear(x, sd["emb_cnn_code.weight"].to(x.dtype), sd["emb_cnn_code.bias"].to(x.dtype))  # model.py:283
    features = F.conv2d(features, sd["emb_features.weight"].to(x.dtype))             # model.py:285-286
    return features, cnn_code


def test_state_dict(enc_sd, seed=0):
    """Weights for the tests: every trunk conv fan-in scaled (normal, std sqrt(2 / fan_in) -- the ReLU gain), BatchNorm
    weight near 1, bias near 0, running statistics near (0, 1), so that activations stay O(1) through all 94 layers
    (checked per layer with ``stats``).  ``enc_sd``: a state_dict giving the keys and shapes."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, v in enc_sd.items():
        if k.endswith("num_batches_tracked"):
            out[k] = torch.zeros_like(v)
        elif k.endswith(".conv.weight"):
            fan = v[0].numel()
            out[k] = torch.randn(v.shape, generator=g) * (2.0 / fan) ** 0.5
        elif k.endswith(".bn.weight"):
            out[k] = 1.0 + 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith(".bn.bias"):
            out[k] = 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith(".running_mean"):
            out[k] = 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith(".running_var"):
            out[k] = 1.0 + 0.2 * torch.rand(v.shape, generator=g)
        elif k == "emb_features.weight":
            out[k] = torch.randn(v.shape, generator=g) * (1.0 / v[0].numel()) ** 0.5
        elif k == "emb_cnn_code.weight":
            out[k] = torch.randn(v.shape, generator=g) * (1.0 / v.shape[1]) ** 0.5
        elif k == "emb_cnn_code.bias":
            out[k] = 0.01 * torch.randn(v.shape, generator=g)
        else:
            raise KeyError(k)
    return out
