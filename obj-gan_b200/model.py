"""Host-side mirror of the reference's module API for the hot path.

Same class names, constructor arguments, ``forward`` signatures and ``state_dict`` keys / shapes as
/root/reference/image_generation/model.py (G side: lines 19-81, 455-795; patch discriminators:
989-1106; object discriminators: 1184-1312) and GlobalAttention.py (73-181), so ``trainer.py`` /
``miscc/losses.py`` call sites stay drop-in and reference checkpoints load with ``strict=True``.
Every forward runs the sm_90a kernels of libobjgan_b200.so through ``ops`` -- no torch.nn compute.

Public tensors are NCHW fp32 exactly like the reference's; internally activations are NHWC with
channels padded to 8 (``*_nhwc`` methods exchange that layout directly and are what G_NET uses
between its stages).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .config import cfg
from .lib import (ACT_LRELU, ACT_NONE, ACT_SIGMOID, ACT_TANH, NA_GLU, NA_LRELU, NA_NONE, PAD_REFLECT, PAD_ZERO,
                  UPSAMPLE2X)
from .ops import cpad


# --------------------------------------------------------------------------------------------------
# parameter holders (leaf modules).  Their attribute names give the reference's state_dict keys.
# --------------------------------------------------------------------------------------------------
# Host-logic tests build dozens of networks on the CPU and never look at the values: they may swap the reference's
# orthogonal initialisation (a QR per weight, seconds for the large layers) for a plain normal draw.
FAST_INIT = False


def _init_weight(w):
    if FAST_INIT:
        w.normal_(0.0, 0.02)
    else:
        nn.init.orthogonal_(w, 1.0)


class Conv2dP(nn.Module):
    """Holds an OIHW ``weight`` (+ optional ``bias``) like nn.Conv2d; forward is an NHWC kernel call."""

    def __init__(self, cin, cout, k, stride=1, pad=1, bias=False, mode=PAD_ZERO, act=ACT_NONE, split=0):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, k, k))
        self.bias = nn.Parameter(torch.empty(cout)) if bias else None
        self.stride, self.pad, self.mode, self.act, self.split = stride, pad, mode, act, split
        self._cache = ops.PackedWeights()
        _init_weight(self.weight.data)
        if bias:
            bound = 1.0 / np.sqrt(cin * k * k)
            nn.init.uniform_(self.bias.data, -bound, bound)

    def forward(self, x):
        return ops.conv2d(x, self.weight, self.bias, self._cache, stride=self.stride, pad=self.pad, mode=self.mode,
                          act=self.act, split=self.split)


class LinearP(nn.Module):
    """nn.Linear parameters ((out, in) weight); runs as a 1x1 conv over a (B, 1, 1, in) tensor."""

    def __init__(self, cin, cout, bias=True, split=0):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin))
        self.bias = nn.Parameter(torch.zeros(cout)) if bias else None
        self.split = split
        self._cache = ops.PackedWeights()
        _init_weight(self.weight.data)

    def forward(self, x2d):
        b = x2d.shape[0]
        w4 = self.weight.view(self.weight.shape[0], self.weight.shape[1], 1, 1)
        y = ops.conv2d(x2d.view(b, 1, 1, -1), w4, self.bias, self._cache, stride=1, pad=0, mode=PAD_ZERO,
                       act=ACT_NONE, split=self.split)
        return y.view(b, -1)


class BatchNormP(nn.Module):
    """nn.BatchNorm{1,2}d parameters/buffers.  Train mode (the trainer never switches G or the Ds to eval():
    trainer.py:331-472) normalises with the batch statistics and updates the running buffers; eval mode (the
    evaluator's netG.eval(), evaluator.py:110) normalises with the running statistics and leaves the buffers alone."""

    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(c).normal_(1.0, 0.02))
        self.bias = nn.Parameter(torch.zeros(c))
        self.register_buffer("running_mean", torch.zeros(c))
        self.register_buffer("running_var", torch.ones(c))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))

    def forward(self, y, act):
        return ops.batch_norm_act(y, self.weight, self.bias,
                                  (self.running_mean, self.running_var, self.num_batches_tracked), act,
                                  training=self.training)


class _Slots(nn.Module):
    """Children registered under the numeric names an nn.Sequential would give them, so that state_dict
    keys match the reference's Sequential-based blocks (parameter-free positions are simply absent)."""

    def __init__(self, **children):
        super().__init__()
        for name, m in children.items():
            self.add_module(name.lstrip("_"), m)

    def __getitem__(self, i):
        return getattr(self, str(i))


def weights_init(m):
    """Mirror of miscc/utils.py:309-319 for this package's parameter holders."""
    if isinstance(m, (Conv2dP, LinearP)):
        _init_weight(m.weight.data)
        if isinstance(m, LinearP) and m.bias is not None:
            m.bias.data.fill_(0.0)
    elif isinstance(m, BatchNormP):
        m.weight.data.normal_(1.0, 0.02)
        m.bias.data.fill_(0)


class _Base(nn.Module):
    def _load_from_state_dict(self, *a, **k):
        ops.bump_param_epoch()
        return super()._load_from_state_dict(*a, **k)


# --------------------------------------------------------------------------------------------------
# blocks
# --------------------------------------------------------------------------------------------------
class GLU(nn.Module):
    """ref: model.py:19-27 (NCHW in / out)."""

    def forward(self, x):
        nc = x.size(1)
        assert nc % 2 == 0, "channels dont divide 2!"
        if x.dim() == 2:
            return ops.glu(x)
        h = nc // 2
        y = ops.to_nhwc(x, nc) if nc % 4 == 0 else None
        assert y is not None
        return ops.to_nchw(ops.glu(y), h)


class UpBlock(_Slots):
    """upBlock (ref: model.py:43-49): keys ``1.weight`` (conv3x3, out*2 channels) and ``2.*`` (BatchNorm2d)."""

    def __init__(self, cin, cout):
        super().__init__(_1=Conv2dP(cin, cout * 2, 3, 1, 1, mode=UPSAMPLE2X, split=cout), _2=BatchNormP(cout * 2))
        assert cout % 8 == 0

    def forward(self, x):
        return self[2](self[1](x), NA_GLU)


def upBlock(in_planes, out_planes):
    return UpBlock(in_planes, out_planes)


class UpBlockIN(_Slots):
    """upBlock(norm=nn.InstanceNorm2d) (ref: model.py:43-49, 910-911): key ``1.weight`` only (the instance norm has no
    parameters)."""

    def __init__(self, cin, cout):
        super().__init__(_1=Conv2dP(cin, cout * 2, 3, 1, 1, mode=UPSAMPLE2X, split=cout))
        assert cout % 8 == 0

    def forward(self, x):  # NHWC
        return ops.instance_norm_act(self[1](x), NA_GLU)


class HmapResBlock(nn.Module):
    """ref: model.py:63-81.  keys ``block.1.weight`` (2C, C, 3, 3) and ``block.5.weight`` (C, C, 3, 3)."""

    def __init__(self, channel_num):
        super().__init__()
        c = channel_num
        self.block = _Slots(_1=Conv2dP(c, 2 * c, 3, 1, 1, mode=PAD_REFLECT, split=c),
                            _5=Conv2dP(c, c, 3, 1, 1, mode=PAD_REFLECT))

    next_pad = None      # set by the owner: halo (1 / 0) of the convolution that consumes this block's output

    def forward(self, x):  # NHWC
        # the GLU output is read by block.5 only: it is written directly as that convolution's fp16 operand copies
        # (reflection halo included) and never as fp32; the block output goes out as fp32 (the next residual add reads
        # it) plus, when the owner said what consumes it, the operand copies of that convolution
        y = ops.instance_norm_act(self.block[1](x), NA_GLU, split_pad=1, keep_f32=False)
        return ops.instance_norm_act(self.block[5](y), NA_NONE, res=x, split_pad=self.next_pad)


def _chain_res_blocks(blocks, last_pad):
    """Tell every block of a residual chain which operand layout its consumer wants: the next block's reflection-padded
    conv (halo 1), or ``last_pad`` for what follows the chain."""
    blocks = list(blocks)
    for b in blocks[:-1]:
        b.next_pad = 1
    if blocks:
        blocks[-1].next_pad = last_pad


class CA_NET(_Base):
    """ref: model.py:455-483.  ``eps`` can be injected (parity tests); otherwise drawn on the device."""

    def __init__(self):
        super().__init__()
        self.t_dim = cfg.TEXT.EMBEDDING_DIM
        self.c_dim = cfg.GAN.CONDITION_DIM
        self.fc = LinearP(self.t_dim, self.c_dim * 4, bias=True, split=self.c_dim * 2)
        self.eps_override = None

    def forward_rows(self, text_embedding):
        """Returns c_code rows (B, cpad(c_dim)) and the GLU output rows x = [mu | logvar | pad]."""
        emb = text_embedding.contiguous()
        assert emb.shape[1] % 8 == 0
        x = ops.glu(self.fc(emb))                      # (B, cpad(2*c_dim))
        eps = self.eps_override
        if eps is None:
            eps = torch.randn(emb.shape[0], self.c_dim, device=emb.device)
        c = ops.reparam(x, eps, self.c_dim)
        return c, x

    def forward(self, text_embedding):
        c, x = self.forward_rows(text_embedding)
        d = self.c_dim
        return c[:, :d], x[:, :d], x[:, d:2 * d]


class INIT_STAGE_G(_Base):
    """ref: model.py:486-518."""

    def __init__(self, ngf, ncf):
        super().__init__()
        self.gf_dim = ngf
        self.in_dim = cfg.GAN.Z_DIM + ncf
        nz = self.in_dim
        self.fc = _Slots(_0=LinearP(nz, ngf * 8 * 8 * 2, bias=False, split=ngf * 8 * 8), _1=BatchNormP(ngf * 8 * 8 * 2))
        self.upsample1 = upBlock(ngf, ngf // 2)
        self.upsample2 = upBlock(ngf // 2, ngf // 4)

    def forward_nhwc(self, z_code, c_rows):
        """z (B, Z) and c_code rows (B, cpad(ncf)) -> (B, 32, 32, ngf/4) NHWC."""
        b = z_code.shape[0]
        ncf = self.in_dim - cfg.GAN.Z_DIM
        cz = ops.cat_channels([c_rows.view(b, 1, 1, -1), z_code.contiguous().view(b, 1, 1, -1)],
                              [ncf, cfg.GAN.Z_DIM])
        y = self.fc[0](cz.view(b, -1))                                  # (B, 2*ngf*64)
        y = self.fc[1](y.view(b, 1, 1, -1), NA_GLU)                      # BatchNorm1d + GLU -> (B,1,1,ngf*64)
        # .view(-1, ngf, 8, 8) of the reference is an NCHW reinterpretation of the feature vector
        x = ops.to_nhwc(y.view(b, self.gf_dim, 8, 8), cpad(self.gf_dim))
        x = self.upsample1(x)
        return self.upsample2(x)

    def forward(self, z_code, c_code):
        b = z_code.shape[0]
        ncf = c_code.shape[1]
        c_rows = torch.zeros(b, cpad(ncf), device=z_code.device)
        c_rows[:, :ncf] = c_code
        return ops.to_nchw(self.forward_nhwc(z_code, c_rows), self.gf_dim // 4)


class G_HMAP(_Base):
    """ref: model.py:589-617.  keys ``conv3x3.1.{weight,bias}``, ``downsample1.0.weight``."""

    def __init__(self, ngf, ncf):
        super().__init__()
        self.gf_dim, self.in_dim = ngf, ncf
        self.conv3x3 = _Slots(_1=Conv2dP(ncf, ngf, 3, 1, 1, bias=True, mode=PAD_REFLECT))
        self.downsample1 = _Slots(_0=Conv2dP(ngf, ngf * 2, 3, 2, 1, act=ACT_LRELU))

    def forward_nhwc(self, hmap_nhwc):
        y = ops.instance_norm_act(self.conv3x3[1](hmap_nhwc), NA_LRELU)
        return self.downsample1[0](y)

    def forward(self, hmap):
        return ops.to_nchw(self.forward_nhwc(ops.to_nhwc(hmap)), self.gf_dim * 2)


class GlobalAttentionGeneral(_Base):
    """ATT_NET (ref: GlobalAttention.py:73-122)."""

    def __init__(self, idf, cdf):
        super().__init__()
        self.conv_context = Conv2dP(cdf, idf, 1, 1, 0)
        self.idf = idf
        self.mask = None

    def applyMask(self, mask):
        self.mask = mask

    def forward_nhwc(self, h_nhwc, context):
        src = ops.words_proj(context, self.conv_context.weight.view(self.idf, -1))
        return ops.att_general(h_nhwc, src, ops.mask_bytes(self.mask), self.idf)

    def forward(self, input, context):
        wc, attn = self.forward_nhwc(ops.to_nhwc(input), context)
        return ops.to_nchw(wc, self.idf), attn


class GlobalBUAttentionGeneral(_Base):
    """BT_ATT_NET (ref: GlobalAttention.py:125-181).  No gradient to the label / GloVe inputs (they are
    data in every caller)."""

    def __init__(self, idf, cdf):
        super().__init__()
        self.conv_context = Conv2dP(cdf, idf, 1, 1, 0)
        self.idf = idf
        self.mask = None
        self.eps = 1e-8

    def applyMask(self, mask):
        self.mask = mask

    def forward(self, input, context1, context2):
        b, e, r = input.shape[0], input.shape[1], input.shape[2] * input.shape[3]
        src = ops.words_proj(context2, self.conv_context.weight.view(self.idf, -1))
        wc, attn = ops.bu_att(input.reshape(b, e, r), context1, src, ops.mask_bytes(self.mask),
                              cfg.TRAIN.BUATTN_NORM)
        return wc.view(b, self.idf, input.shape[2], input.shape[3]), attn.view(b, -1, input.shape[2], input.shape[3])


ATT_NET = GlobalAttentionGeneral
BT_ATT_NET = GlobalBUAttentionGeneral


def pprocess_bt_attns(fmaps, ih, iw, bt_mask):
    """ref: miscc/utils.py:401-413.  Accepts the reference's expanded (B, R, num, ih, iw) mask or the compact
    (B, R, ih, iw) one; returns NCHW (B, num, ih, iw)."""
    if bt_mask.dim() == 5:
        bt_mask = bt_mask[:, :, 0]
    b, num, r = fmaps.shape[0], fmaps.shape[1], fmaps.shape[2]
    out = ops.paint_max(fmaps.reshape(b, num, r), bt_mask[:, :r].contiguous())
    return ops.to_nchw(out, num)


def _bt_branch(bt_att, slabels_feat, glove_word_embs, word_embs, mask, bt_mask, ef_dim2):
    """Shared by the INIT / NEXT stage mains (ref: model.py:552-569, 668-687)."""
    rmax = slabels_feat.shape[2]
    if rmax == 0:
        # ref: model.py:571-576 / 689-694 -- a batch without boxes contributes all-zero code / attention / label maps
        # (the reference's INIT-stage `else` reads an undefined `att`; its intent, zeros, is what the NEXT stage does)
        b, (ih, iw) = slabels_feat.shape[0], bt_mask.shape[2:]
        z = lambda c: torch.zeros((b, ih, iw, ops.cpad(c)), device=bt_mask.device, dtype=torch.float32)
        raw = torch.zeros((b, bt_att.idf, 0, 1), device=bt_mask.device, dtype=torch.float32)
        return raw, z(bt_att.idf), z(mask.shape[1]), z(ef_dim2)
    bt_att.applyMask(mask)
    bt_c_code, bt_att_map = bt_att(slabels_feat, glove_word_embs, word_embs)          # (B,idf,R,1), (B,L,R,1)
    b = bt_c_code.shape[0]
    m = bt_mask[:, :rmax].contiguous()
    code_nhwc = ops.paint_max(bt_c_code.reshape(b, -1, rmax), m)
    att_nhwc = ops.paint_max(bt_att_map.reshape(b, -1, rmax), m)
    slab_nhwc = ops.paint_max(slabels_feat.reshape(b, ef_dim2, rmax), m)
    return bt_c_code, code_nhwc, att_nhwc, slab_nhwc


class INIT_STAGE_G_MAIN(_Base):
    """ref: model.py:521-586."""

    def __init__(self, ngf, nef, nef2):
        super().__init__()
        self.gf_dim, self.ef_dim, self.ef_dim2 = ngf, nef, nef2
        self.bt_att = BT_ATT_NET(ngf, nef)
        c = ngf * 3 + nef2
        self.residual = nn.Sequential(*[HmapResBlock(c) for _ in range(cfg.GAN.GLB_R_NUM)])
        self.upsample = upBlock(c, ngf)
        _chain_res_blocks(self.residual, 0)          # the upsample conv reads the plain (halo-free) operand copies

    def forward_nhwc(self, h_code_hmap, h_code1_sent, word_embs, glove_word_embs, slabels_feat, mask, bt_mask):
        ngf = self.gf_dim
        # max_num_roi comes from slabels_feat's third dim (the trainer builds it with max(num_rois) slots,
        # miscc/utils.py:502-522), so no device->host sync on num_rois is needed here.
        _, code, _att, slab = _bt_branch(self.bt_att, slabels_feat, glove_word_embs, word_embs, mask, bt_mask,
                                         self.ef_dim2)
        x = ops.cat_channels([h_code_hmap, h_code1_sent, code, slab], [ngf, ngf, ngf, self.ef_dim2])
        x = self.residual(x)
        return self.upsample(x)

    def forward(self, h_code_hmap, h_code1_sent, c_code, word_embs, glove_word_embs, slabels_feat, mask, rois,
                num_rois, bt_mask, glb_max_num_roi):
        rmax = int(np.amax(num_rois.data.cpu().numpy()))
        out = self.forward_nhwc(ops.to_nhwc(h_code_hmap), ops.to_nhwc(h_code1_sent), word_embs, glove_word_embs,
                                slabels_feat[:, :, :rmax], mask, bt_mask)
        return ops.to_nchw(out, self.gf_dim)


class NEXT_STAGE_G_MAIN(_Base):
    """ref: model.py:620-705."""

    def __init__(self, ngf, nef, nef2):
        super().__init__()
        self.gf_dim, self.ef_dim, self.ef_dim2 = ngf, nef, nef2
        self.att = ATT_NET(ngf, nef)
        self.bt_att = BT_ATT_NET(ngf, nef)
        c = ngf * 3 + nef2
        self.residual = nn.Sequential(*[HmapResBlock(c) for _ in range(cfg.GAN.LOCAL_R_NUM)])
        self.upsample = upBlock(c, ngf)
        _chain_res_blocks(self.residual, 0)

    def forward_nhwc(self, h_code, h_code_hmap, word_embs, glove_word_embs, slabels_feat, mask, bt_mask,
                     glb_max_num_roi):
        ngf = self.gf_dim
        self.att.applyMask(mask)
        c_code, att = self.att.forward_nhwc(h_code, word_embs)
        raw, code, bt_att, slab = _bt_branch(self.bt_att, slabels_feat, glove_word_embs, word_embs, mask, bt_mask,
                                             self.ef_dim2)
        b, rmax = raw.shape[0], raw.shape[2]
        raw_full = raw.new_zeros(b, ngf, glb_max_num_roi, 1)
        raw_full[:, :, :rmax] = raw
        x = ops.cat_channels([ops.add(h_code, h_code_hmap), c_code, code, slab], [ngf, ngf, ngf, self.ef_dim2])
        x = self.residual(x)
        out = self.upsample(x)
        return out, raw_full.transpose(1, 2).squeeze(-1), att, bt_att

    def forward(self, h_code, h_code_hmap, c_code, word_embs, glove_word_embs, slabels_feat, mask, rois, num_rois,
                bt_mask, glb_max_num_roi):
        rmax = int(np.amax(num_rois.data.cpu().numpy()))
        out, raw, att, bt_att = self.forward_nhwc(ops.to_nhwc(h_code), ops.to_nhwc(h_code_hmap), word_embs,
                                                  glove_word_embs, slabels_feat[:, :, :rmax], mask, bt_mask,
                                                  glb_max_num_roi)
        L = att.shape[1]
        return ops.to_nchw(out, self.gf_dim), raw, att, ops.to_nchw(bt_att, L)


class GET_IMAGE_G(_Base):
    """ref: model.py:708-719.  key ``img.0.weight``."""

    def __init__(self, ngf):
        super().__init__()
        self.gf_dim = ngf
        self.img = _Slots(_0=Conv2dP(ngf, 3, 3, 1, 1, act=ACT_TANH))

    def forward_nhwc(self, h):
        return self.img[0](h)

    def forward(self, h_code):
        return ops.to_nchw(self.forward_nhwc(ops.to_nhwc(h_code)), 3)


class G_NET(_Base):
    """ref: model.py:722-795 -- same forward signature and return tuple."""

    def __init__(self, num_classes):
        super().__init__()
        ngf, nef, nef2, ncf = cfg.GAN.GF_DIM, cfg.TEXT.EMBEDDING_DIM, cfg.TEXT.GLOVE_EMBEDDING_DIM, cfg.GAN.CONDITION_DIM
        self.ca_net = CA_NET()
        self.num_classes = num_classes
        self.branch_num = cfg.TREE.BRANCH_NUM
        if cfg.TREE.BRANCH_NUM > 0:
            self.h_net1_sent = INIT_STAGE_G(ngf * 4, ncf)
            self.h_net1_hmap = G_HMAP(ngf // 2, num_classes)
            self.h_net1_main = INIT_STAGE_G_MAIN(ngf, nef, nef2)
            self.img_net1 = GET_IMAGE_G(ngf)
        if cfg.TREE.BRANCH_NUM > 1:
            self.h_net2_hmap = G_HMAP(ngf // 2, num_classes)
            self.h_net2_main = NEXT_STAGE_G_MAIN(ngf, nef, nef2)
            self.img_net2 = GET_IMAGE_G(ngf)
        if cfg.TREE.BRANCH_NUM > 2:
            self.h_net3_hmap = G_HMAP(ngf // 2, num_classes)
            self.h_net3_main = NEXT_STAGE_G_MAIN(ngf, nef, nef2)
            self.img_net3 = GET_IMAGE_G(ngf)

    def forward(self, z_code, sent_emb, word_embs, glove_word_embs, slabels_feat, mask, hmaps, rois, fm_rois,
                num_rois, bt_masks, fm_bt_masks, glb_max_num_roi):
        fake_imgs, bt_c_codes, att_maps, bt_att_maps = [], [], [], []
        c_rows, x_rows = self.ca_net.forward_rows(sent_emb)
        d = self.ca_net.c_dim
        mu, logvar = x_rows[:, :d], x_rows[:, d:2 * d]
        self._ca_rows = x_rows            # [mu | logvar | pad] rows for the fused KL kernel (losses.KL_loss)
        words = word_embs.contiguous()
        glove = glove_word_embs.contiguous()
        L = words.shape[2]
        h = None
        if self.branch_num > 0:
            hh = self.h_net1_hmap.forward_nhwc(ops.to_nhwc(hmaps[0]))
            hs = self.h_net1_sent.forward_nhwc(z_code, c_rows)
            h = self.h_net1_main.forward_nhwc(hh, hs, words, glove, slabels_feat, mask, fm_bt_masks)
            fake_imgs.append(ops.to_nchw(self.img_net1.forward_nhwc(h), 3))
        for k in range(2, self.branch_num + 1):
            hmap_net = getattr(self, f"h_net{k}_hmap")
            main = getattr(self, f"h_net{k}_main")
            hh = hmap_net.forward_nhwc(ops.to_nhwc(hmaps[k - 1]))
            h, raw, att, bt_att = main.forward_nhwc(h, hh, words, glove, slabels_feat, mask, bt_masks[k - 2],
                                                    glb_max_num_roi)
            fake_imgs.append(ops.to_nchw(getattr(self, f"img_net{k}").forward_nhwc(h), 3))
            bt_c_codes.append(raw)
            att_maps.append(att)
            bt_att_maps.append(ops.to_nchw(bt_att, L))
        return fake_imgs, bt_c_codes, att_maps, bt_att_maps, mu, logvar


# --------------------------------------------------------------------------------------------------
# shape generator (ref: model.py:798-985): one soft mask per roi slot from the layout's box maps.  Inference only.
# --------------------------------------------------------------------------------------------------
class _DownBlock3x3(_Slots):
    """downBlock_3x3 (ref: model.py:800-806): conv3x3 stride 2, no bias -> InstanceNorm2d -> LeakyReLU(0.2)."""

    def __init__(self, cin, cout):
        super().__init__(_0=Conv2dP(cin, cout, 3, 2, 1))

    def forward(self, x):  # NHWC
        return ops.instance_norm_act(self[0](x), NA_LRELU)


class CLSTMCell(_Base):
    """ref: model.py:818-863.  key ``Gates.{weight,bias}``: conv over cat(x_t, h_{t-1}).  Run by SHP_G_NET as two
    convolutions split by input channels: the x-part (with the bias) once for all steps, the h-part inside the loop
    (skipped at t = 0, where h = 0).  The split copies are derived from ``Gates.weight`` and refreshed whenever it
    changes (load_state_dict, in-place edits)."""

    def __init__(self, input_size, hidden_size, kernel_size, padding):
        super().__init__()
        self.input_size, self.hidden_size = input_size, hidden_size
        self.Gates = Conv2dP(input_size + hidden_size, 4 * hidden_size, kernel_size, 1, padding, bias=True)
        self._split_key = None
        self._wx = self._wh = None
        self._caches = (ops.PackedWeights(), ops.PackedWeights())

    def split_weights(self):
        w = self.Gates.weight
        key = (w.data_ptr(), w._version, ops._epoch_of(w))
        if key != self._split_key:
            ci = self.input_size
            if self._wx is None or self._wx.device != w.device:
                self._wx = torch.empty_like(w[:, :ci]).contiguous()
                self._wh = torch.empty_like(w[:, ci:]).contiguous()
            self._wx.copy_(w.detach()[:, :ci])          # bumps _version: the packed operand copies are rebuilt
            self._wh.copy_(w.detach()[:, ci:])
            self._split_key = key
        return self._wx, self._wh

    def gates_x(self, x):
        """x-part of Gates plus its bias: NHWC (N, H, W, input_size) -> (N, H, W, 4 * hidden_size)."""
        return ops.conv2d(x, self.split_weights()[0], self.Gates.bias, self._caches[0], stride=1, pad=self.Gates.pad)

    def gates_h(self, h):
        """h-part of Gates (no bias): NHWC (N, H, W, hidden_size) -> (N, H, W, 4 * hidden_size)."""
        return ops.conv2d(h, self.split_weights()[1], None, self._caches[1], stride=1, pad=self.Gates.pad)


class ShapeResBlock(nn.Module):
    """ResBlock(channel_num, norm=nn.InstanceNorm2d) (ref: model.py:866-882): keys ``block.{0,3,6}.weight``; zero
    padding, and no norm after the last convolution."""

    def __init__(self, channel_num):
        super().__init__()
        c = channel_num
        self.block = _Slots(_0=Conv2dP(c, 2 * c, 3, 1, 1, split=c), _3=Conv2dP(c, 2 * c, 3, 1, 1, split=c),
                            _6=Conv2dP(c, c, 3, 1, 1))

    def forward(self, x):  # NHWC
        y = ops.instance_norm_act(self.block[0](x), NA_GLU)
        y = ops.instance_norm_act(self.block[3](y), NA_GLU)
        return ops.add(self.block[6](y), x)


class GET_SHAPE_G(nn.Module):
    """ref: model.py:885-895.  key ``img.0.weight``: conv1x1 nbf -> 1, no bias, sigmoid."""

    def __init__(self, nbf):
        super().__init__()
        self.img = _Slots(_0=Conv2dP(nbf, 1, 1, 1, 0, act=ACT_SIGMOID))

    def forward_nhwc(self, h):
        return self.img[0](h)


class SHP_G_NET(_Base):
    """ref: model.py:898-985 -- same constructor, forward signature and state_dict.  Inference only: a forward with grad
    mode on and parameters that require grad raises."""

    def __init__(self, num_classes):
        super().__init__()
        nbf = num_classes
        self.nbf = nbf
        self.fm_size = cfg.ROI.FM_SIZE
        self.downsample1 = _DownBlock3x3(nbf, nbf * 2)
        self.downsample2 = _DownBlock3x3(nbf * 2, nbf * 4)
        self.fwd_convlstm = CLSTMCell(nbf * 4, nbf * 2, 3, 1)
        self.bwd_convlstm = CLSTMCell(nbf * 4, nbf * 2, 3, 1)
        self.jointConv = _Slots(_0=Conv2dP(nbf * 8, nbf * 8, 3, 1, 1, split=nbf * 4))
        self.residual = nn.Sequential(*[ShapeResBlock(nbf * 4) for _ in range(cfg.GAN.R_NUM)])
        self.upsample1 = UpBlockIN(nbf * 4, nbf * 2)
        self.upsample2 = UpBlockIN(nbf * 2, nbf)
        self.img_net = GET_SHAPE_G(nbf)

    def _check_inference(self, *inputs):
        ops.inference_only("SHP_G_NET", *inputs, *self.parameters())

    def forward_nhwc(self, z_code, maps, bbox_fmaps):
        """z_code (B, R, 4*nbf); maps NHWC (2*B*R, S, S, cpad(nbf)): the forward sequence (image b*R + t), then the
        backward one (what ops.form_bbox_maps builds); bbox_fmaps (B, R, F, F).  Returns the masks as NHWC
        (B*R, S, S, 8), channel 0 (the conv head's padded output)."""
        self._check_inference(z_code, maps, bbox_fmaps)
        b, r = z_code.shape[0], z_code.shape[1]
        n = b * r
        if n == 0:
            return torch.zeros((0, maps.shape[1], maps.shape[2], 8), device=maps.device, dtype=torch.float32)
        h = self.downsample2(self.downsample1(maps))               # both sequences in one pass: (2BR, F, F, 4*nbf)
        gx = (self.fwd_convlstm.gates_x(h[:n]), self.bwd_convlstm.gates_x(h[n:]))
        fm, ch, cz = h.shape[1], self.nbf * 2, self.nbf * 4
        joint = torch.empty((n, fm, fm, 2 * ch + cz), device=h.device, dtype=torch.float32)
        ops.fill_channels(joint, z_code.reshape(n, cz), 2 * ch)  # z broadcast over the map (model.py:931-935, 962)
        c = (torch.empty((b, fm, fm, ch), device=h.device, dtype=torch.float32),
             torch.empty((b, fm, fm, ch), device=h.device, dtype=torch.float32))
        hs = None
        for t in range(r):
            gh = None if t == 0 else (self.fwd_convlstm.gates_h(hs[0]), self.bwd_convlstm.gates_h(hs[1]))
            hs = ops.clstm_cell(gx, gh, c, joint, t)
        y = ops.instance_norm_act(self.jointConv[0](joint), NA_GLU)
        y = ops.mul_pixels(y, bbox_fmaps)                            # crop (model.py:969-972)
        y = self.residual(y)
        y = self.upsample2(self.upsample1(y))
        return self.img_net.forward_nhwc(y)

    def forward(self, z_code, bbox_maps_fwd, bbox_maps_bwd, bbox_fmaps):
        """NCHW like the reference: z_code (B, R, 4*nbf), bbox_maps_* (B, R, nbf, S, S), bbox_fmaps (B, R, F, F) ->
        (B, R, 1, S, S)."""
        self._check_inference(z_code, bbox_maps_fwd, bbox_maps_bwd, bbox_fmaps)
        b, r = z_code.shape[0], z_code.shape[1]
        s = bbox_maps_fwd.shape[-1]
        maps = ops.nchw_rows([bbox_maps_fwd.reshape(b * r, self.nbf, s, s), bbox_maps_bwd.reshape(b * r, self.nbf, s, s)],
                             cpad(self.nbf))
        out = self.forward_nhwc(z_code.contiguous(), maps, bbox_fmaps.contiguous())
        return ops.to_nchw(out, 1).view(b, r, 1, s, s)


# --------------------------------------------------------------------------------------------------
# text encoder
# --------------------------------------------------------------------------------------------------
class _EmbeddingP(nn.Module):
    """nn.Embedding's ``weight`` (ntoken, ninput), initialised like RNN_ENCODER.init_weights (model.py:125-127)."""

    def __init__(self, ntoken, ninput):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(ntoken, ninput).uniform_(-0.1, 0.1))


class _BiLSTMP(nn.Module):
    """One-layer bidirectional nn.LSTM's parameters, in its state_dict order and with its initialisation."""

    def __init__(self, ninput, nhidden):
        super().__init__()
        k = 1.0 / np.sqrt(nhidden)
        for sfx in ("", "_reverse"):
            for name, shape in (("weight_ih", (4 * nhidden, ninput)), ("weight_hh", (4 * nhidden, nhidden)),
                                ("bias_ih", (4 * nhidden,)), ("bias_hh", (4 * nhidden,))):
                self.register_parameter(f"{name}_l0{sfx}", nn.Parameter(torch.empty(shape).uniform_(-k, k)))


class RNN_ENCODER(_Base):
    """ref: model.py:85-179 -- same constructor, state_dict keys / shapes and ``forward(captions, cap_lens, max_len)``
    -> (words_emb (B, nhidden, max_len), sent_emb (B, nhidden)).  Inference only (the reference always runs it after
    .eval(): trainer.py:100, evaluator.py:95): dropout is not implemented, so a forward in training mode raises, and so
    does one with grad mode on and parameters that require grad.  One-layer bidirectional LSTM only.

    The batch need not be sorted by length: each sample runs its own cap_lens[b] steps, with results bitwise
    independent of its place in the batch.  The forward is three library calls -- the token lookup
    (og_gather_rows from a channel-padded copy of ``encoder.weight``), the x-part of the gates of both directions for
    every step (one 1x1 og_conv2d_simt with bias b_ih + b_hh) and the recurrence (og_lstm_bidir) -- and reads no
    lengths on the host.  The padded copies are derived from the parameters and refreshed whenever they change."""

    def __init__(self, ntoken, ninput=300, drop_prob=0.5, nhidden=128, nlayers=1, bidirectional=True):
        super().__init__()
        if cfg.RNN_TYPE != "LSTM" or nlayers != 1 or not bidirectional:
            raise NotImplementedError("RNN_ENCODER supports the one-layer bidirectional LSTM only")
        self.n_steps = cfg.TEXT.WORDS_NUM
        self.ntoken, self.ninput, self.drop_prob = ntoken, ninput, drop_prob
        self.nlayers, self.bidirectional, self.rnn_type = nlayers, bidirectional, cfg.RNN_TYPE
        self.num_directions = 2
        self.nhidden = nhidden // self.num_directions
        self.encoder = _EmbeddingP(ntoken, ninput)
        self.rnn = _BiLSTMP(ninput, self.nhidden)
        self._derived_key = None
        self._emb = self._wih = self._bias = None
        self._cache = ops.PackedWeights()

    def _params_key(self):
        ps = list(self.parameters())
        return tuple((p.data_ptr(), p._version) for p in ps) + (ops._epoch_of(ps[0]),)

    def derived_weights(self):
        """(encoder.weight padded to cpad(ninput) channels, W_ih of both directions as a (8H, ninput, 1, 1) conv weight,
        b_ih + b_hh of both directions (8H,)), rebuilt when a parameter changes, in place (stable addresses)."""
        key = self._params_key()
        if key != self._derived_key:
            w, r = self.encoder.weight, self.rnn
            dev, cp, g = w.device, cpad(self.ninput), 4 * self.nhidden
            if self._emb is None or self._emb.device != dev:
                self._emb = torch.empty((self.ntoken, cp), device=dev, dtype=torch.float32)
                self._wih = torch.empty((2 * g, self.ninput, 1, 1), device=dev, dtype=torch.float32)
                self._bias = torch.empty((2 * g,), device=dev, dtype=torch.float32)
            ops.zeros_into(self._emb)
            ops.copy_channels(w.detach(), self.ninput, self._emb, cp, self.ntoken)
            wih = self._wih.view(2 * g, self.ninput)
            wih[:g].copy_(r.weight_ih_l0.detach())
            wih[g:].copy_(r.weight_ih_l0_reverse.detach())
            ops.add_into(r.bias_ih_l0, r.bias_hh_l0, self._bias[:g])
            ops.add_into(r.bias_ih_l0_reverse, r.bias_hh_l0_reverse, self._bias[g:])
            self._derived_key = self._params_key()
        return self._emb, self._wih, self._bias

    def _check_inference(self, *inputs):
        if self.training:
            raise RuntimeError("RNN_ENCODER is inference only and has no dropout: call .eval() first")
        ops.inference_only("RNN_ENCODER", *inputs, *self.parameters())

    def forward(self, captions, cap_lens, max_len, mask=None):
        """captions (B, >= max_len) int64 token ids, cap_lens (B,) int64 in [1, max_len] (device tensors; not read on
        the host), max_len: the words_emb width (the reference passes max(cap_lens))."""
        self._check_inference()
        gx, max_len = self._gate_inputs(captions, cap_lens, max_len)
        return ops.lstm_bidir(gx, self.rnn.weight_hh_l0, self.rnn.weight_hh_l0_reverse, cap_lens, max_len)

    def _gate_inputs(self, captions, cap_lens, max_len):
        """The x-part of the gates of both directions for the first max_len tokens: (B*max_len, 8H), max_len."""
        b, max_len = captions.shape[0], int(max_len)
        assert captions.shape[1] >= max_len and cap_lens.shape == (b,)
        emb, wih, bias = self.derived_weights()
        ids = captions[:, :max_len]
        ids = ids if ids.is_contiguous() else ids.contiguous()
        x = ops.gather_rows(emb, ids.reshape(-1))                                     # (B*L, cpad(ninput))
        return ops.linear_rows(x, wih, bias, self._cache), max_len                    # (B*L, 8H)


class PreEncoderRNN(RNN_ENCODER):
    """The box generator's caption encoder (ref: box_generation/seq2seq/models/PreEncoderRNN.py:6-99) -- the same
    constructor, state_dict keys and shapes, and ``forward(captions, cap_lens)`` -> (output (B, T, 2H), (h_n, c_n)),
    h_n / c_n (2, B, H), T = max(cap_lens).  The reference builds it with nhidden=256 and loads the image side's
    text_encoder100.pth (sample.py:179-182), so it is RNN_ENCODER's network and shares its gate-input path; the
    recurrence also returns the final cell state (og_lstm_bidir_state).  Inference only, like RNN_ENCODER; one-layer
    bidirectional LSTM with nhidden=256 only.  Captions of any length are read in full (the box path does not truncate
    them to WORDS_NUM); the recurrence has no length limit and is tested to 64 tokens."""

    def __init__(self, ntoken, ninput=300, drop_prob=0.5, nhidden=128, nlayers=1, bidirectional=True):
        if nhidden != 256 or nlayers != 1 or not bidirectional:
            raise NotImplementedError("PreEncoderRNN supports the one-layer bidirectional LSTM with nhidden=256 only")
        _Base.__init__(self)
        self.ntoken, self.ninput, self.drop_prob = ntoken, ninput, drop_prob
        self.nlayers, self.bidirectional, self.rnn_type = nlayers, bidirectional, "LSTM"
        self.num_directions = 2
        self.nhidden = nhidden // self.num_directions
        self.encoder = _EmbeddingP(ntoken, ninput)
        self.rnn = _BiLSTMP(ninput, self.nhidden)
        self._derived_key = None
        self._emb = self._wih = self._bias = None
        self._cache = ops.PackedWeights()

    def encode_state(self, captions, cap_lens, max_len):
        """(words (B, 2H, max_len), h (B, 2H), c (B, 2H)): the state with its directions concatenated, as the decoder
        reads it (DecoderRNN._cat_directions).  cap_lens is not read on the host."""
        self._check_inference()
        gx, max_len = self._gate_inputs(captions, cap_lens, max_len)
        return ops.lstm_bidir_state(gx, self.rnn.weight_hh_l0, self.rnn.weight_hh_l0_reverse, cap_lens, max_len)

    def forward(self, captions, cap_lens):
        cap_lens = torch.as_tensor(cap_lens, dtype=torch.int64, device=captions.device)
        words, h, c = self.encode_state(captions, cap_lens, int(cap_lens.max()))   # pad_packed_sequence's width
        b, hid = captions.shape[0], self.nhidden
        return words.transpose(1, 2), (h.view(b, 2, hid).transpose(0, 1), c.view(b, 2, hid).transpose(0, 1))


class _LinearP(nn.Module):
    """nn.Linear's ``weight`` / ``bias``."""

    def __init__(self, fin, fout):
        super().__init__()
        k = 1.0 / np.sqrt(fin)
        self.weight = nn.Parameter(torch.empty(fout, fin).uniform_(-k, k))
        self.bias = nn.Parameter(torch.empty(fout).uniform_(-k, k))


class _LSTMP(nn.Module):
    """One-layer unidirectional nn.LSTM's parameters."""

    def __init__(self, ninput, nhidden):
        super().__init__()
        k = 1.0 / np.sqrt(nhidden)
        for name, shape in (("weight_ih", (4 * nhidden, ninput)), ("weight_hh", (4 * nhidden, nhidden)),
                            ("bias_ih", (4 * nhidden,)), ("bias_hh", (4 * nhidden,))):
            self.register_parameter(f"{name}_l0", nn.Parameter(torch.empty(shape).uniform_(-k, k)))


class DecoderRNN(_Base):
    """The box decoder (ref: box_generation/seq2seq/models/DecoderRNN.py:21-79) -- the same constructor, state_dict
    keys and shapes -- and its inference branch (:260-292) as ``sample``.  Inference only (the reference samples after
    .eval(), sample.py:165): a sample in training mode raises, and so does one with grad mode on and parameters that
    require grad.  The attention variant, the GRU cell, more than one layer, and any hidden size but 256 or mixture size
    but 5 raise NotImplementedError."""

    def __init__(self, l_word2index, x_mean, y_mean, w_mean, r_mean, batch_size, max_len, hidden_size, gmm_comp_num,
                 n_layers=1, rnn_cell="lstm", bidirectional=False, input_dropout_p=0, dropout_p=0, use_attention=False):
        super().__init__()
        if use_attention or str(rnn_cell).lower() != "lstm" or n_layers != 1 or hidden_size != 256 or \
                gmm_comp_num != 5 or not bidirectional:
            raise NotImplementedError("DecoderRNN supports the one-layer LSTM decoder without attention (hidden_size "
                                      "256, 5 mixture components) on a bidirectional encoder only")
        self.l_word2index = dict(l_word2index)
        self.l_output_size = len(l_word2index)
        if self.l_output_size > 128:
            raise NotImplementedError("DecoderRNN supports at most 128 labels")
        self.l_sos_id, self.l_eos_id = l_word2index["<sos>"], l_word2index["<eos>"]
        self.x_mean, self.y_mean, self.w_mean, self.r_mean = x_mean, y_mean, w_mean, r_mean
        self.batch_size, self.max_length, self.hidden_size = batch_size, max_len, hidden_size
        self.gmm_comp_num, self.n_layers, self.bidirectional_encoder = gmm_comp_num, n_layers, bidirectional
        self.input_dropout_p, self.dropout_p, self.use_attention = input_dropout_p, dropout_p, use_attention
        self.aug_size = 50
        nl, h, aug = self.l_output_size, hidden_size, self.aug_size
        self.l_embedding = _EmbeddingP(nl, h)
        self.xy_embedding = _LinearP(2, aug)
        self.wh_embedding = _LinearP(2, aug)
        self.next_xy_embedding = _LinearP(2, aug)
        self.rnn = _LSTMP(h + 2 * aug, h)
        self.l_out = _LinearP(h, nl)
        self.xy_out = _LinearP(h + nl, 6 * gmm_comp_num)
        self.wh_out = _LinearP(h + nl + aug, 6 * gmm_comp_num)
        self._derived_key = None
        self._packed = None

    def _params_key(self):
        ps = list(self.parameters())
        return tuple((p.data_ptr(), p._version) for p in ps) + (ops._epoch_of(ps[0]),)

    def packed_weights(self) -> dict:
        """The kernel-native copies og_box_decode reads (ops.BOX_PACKED), rebuilt in place when a parameter changes:
        the label table (og_box_label_table), the transposed [xy | wh] columns of W_ih with W_hh, and the transposed
        heads."""
        key = self._params_key()
        if key != self._derived_key:
            r = self.rnn
            w = {"wt": torch.cat([r.weight_ih_l0[:, :2 * self.aug_size], r.weight_hh_l0], 1).t(),
                 "lout_t": self.l_out.weight.t(), "xyo_t": self.xy_out.weight.t(), "who_t": self.wh_out.weight.t(),
                 "lout_b": self.l_out.bias, "xyo_b": self.xy_out.bias, "who_b": self.wh_out.bias}
            for k, m in (("xy", self.xy_embedding), ("wh", self.wh_embedding), ("nxy", self.next_xy_embedding)):
                w[k + "_w"], w[k + "_b"] = m.weight, m.bias
            if self._packed is None or self._packed["wt"].device != r.weight_hh_l0.device:
                self._packed = {k: torch.empty(v.shape, device=v.device, dtype=torch.float32) for k, v in w.items()}
                self._packed["table"] = torch.empty((self.l_output_size, 4 * self.hidden_size),
                                                    device=r.weight_hh_l0.device, dtype=torch.float32)
            with torch.no_grad():
                for k, v in w.items():
                    self._packed[k].copy_(v)
                self._packed["table"].copy_(ops.box_label_table(self.l_embedding.weight, r.weight_ih_l0, r.bias_ih_l0,
                                                                r.bias_hh_l0))
            self._derived_key = self._params_key()
        return self._packed

    def _check_inference(self, *inputs):
        if self.training:
            raise RuntimeError("DecoderRNN is inference only and has no dropout: call .eval() first")
        ops.inference_only("DecoderRNN", *inputs, *self.parameters())

    def sample_state(self, h0, c0, noise, early_stop_len, debug=False):
        """``sample`` on the concatenated state h0 / c0 (B, 256)."""
        self._check_inference(h0, c0)
        return ops.box_decode(h0, c0, self.packed_weights(), noise, int(early_stop_len), self.l_sos_id, self.l_eos_id,
                              (self.x_mean, self.y_mean, self.w_mean, self.r_mean), debug)

    def sample(self, encoder_hidden, noise, early_stop_len=10, debug=False):
        """The inference branch for every sample of the batch at once, each stopping after its own <eos> step or after
        early_stop_len steps.  encoder_hidden: (h_n, c_n), each (2, B, 128) (PreEncoderRNN's); noise (B, >=
        early_stop_len, 6): per step (u_xy, n1, n2, u_wh, n3, n4), two uniforms in [0, 1) for the component choices and
        four standard normals.  Returns labels (B, S) int64 (-1 after the end), the normalised samples (B, S, 4) (x, y,
        w, r), the steps taken (B,) and, with debug, (B, S, n_labels + 60): each step's p and both mixture parameter
        sets (pi, mu_x, mu_y, sigma_x, sigma_y, rho)."""
        h_n, c_n = encoder_hidden
        b = h_n.shape[1]
        cat = lambda t: t.transpose(0, 1).reshape(b, 2 * t.shape[2])     # _cat_directions
        return self.sample_state(cat(h_n), cat(c_n), noise, early_stop_len, debug)


# --------------------------------------------------------------------------------------------------
# discriminators
# --------------------------------------------------------------------------------------------------
class _EncodeImage(nn.Module):
    """encode_image_by_ntimes (ref: model.py:999-1017): keys ``0.weight``, then ``{2,5,8}.weight`` convs and
    ``{3,6,9}.*`` BatchNorm2d."""

    def __init__(self, ngf, ndf, n_layer):
        super().__init__()
        self.add_module("0", Conv2dP(3 + ngf, ndf, 4, 2, 1, act=ACT_LRELU))
        self.n_layer = n_layer
        for n in range(1, n_layer):
            prev, cur = ndf * min(2 ** (n - 1), 8), ndf * min(2 ** n, 8)
            i = 2 + 3 * (n - 1)
            self.add_module(str(i), Conv2dP(prev, cur, 4, 2, 1))
            self.add_module(str(i + 1), BatchNormP(cur))

    def forward(self, x):  # NHWC
        x = getattr(self, "0")(x)
        for n in range(1, self.n_layer):
            i = 2 + 3 * (n - 1)
            x = getattr(self, str(i + 1))(getattr(self, str(i))(x), NA_LRELU)
        return x


class D_GET_LOGITS(_Base):
    """ref: model.py:1020-1048.  keys ``jointConv.0.weight``, ``jointConv.1.*``, ``outlogits.0.{weight,bias}``.
    ``forward`` takes / returns NCHW like the reference; ``forward_nhwc`` takes the NHWC feature map."""

    def __init__(self, ndf, nef, bcondition=False):
        super().__init__()
        self.df_dim, self.ef_dim, self.bcondition = ndf, nef, bcondition
        self.layer_num = cfg.GAN.LAYER_D_NUM
        c = ndf * pow(2, self.layer_num - 1)
        if bcondition:
            self.jointConv = _Slots(_0=Conv2dP(c + nef, c, 3, 1, 1), _1=BatchNormP(c))
        self.outlogits = _Slots(_0=Conv2dP(c, 1, 4, 2, 0, bias=True, act=ACT_SIGMOID))

    def forward_nhwc(self, h, c_code=None):
        if self.bcondition and c_code is not None:
            hc = ops.broadcast_cat(h, c_code.reshape(-1, self.ef_dim))
            h = self.jointConv[1](self.jointConv[0](hc), NA_LRELU)
        return ops.to_nchw(self.outlogits[0](h), 1)

    def forward(self, h_code, c_code=None):
        if isinstance(h_code, NHWCFeature):
            return self.forward_nhwc(h_code.t, c_code)
        return self.forward_nhwc(ops.to_nhwc(h_code), c_code)


class NHWCFeature:
    """Feature map handed from a D body to its logit heads without a layout round trip.  Behaves like the
    NCHW tensor the reference returns for the few things callers do with it (``size(0)``, batch slicing:
    miscc/losses.py:185-190); ``.nchw()`` materialises the reference layout."""

    def __init__(self, t, c):
        self.t, self.c = t, c

    def size(self, dim=None):
        n, h, w, _ = self.t.shape
        s = torch.Size((n, self.c, h, w))
        return s if dim is None else s[dim]

    @property
    def shape(self):
        return self.size()

    def __getitem__(self, idx):
        assert isinstance(idx, slice), "only batch slicing is supported on an NHWC feature handle"
        return NHWCFeature(self.t[idx], self.c)

    def nchw(self):
        return ops.to_nchw(self.t, self.c)


class _PatD(_Base):
    def __init__(self, b_jcu=True):
        super().__init__()
        ndf, nef = cfg.GAN.DF_DIM, cfg.TEXT.EMBEDDING_DIM
        self.img_code = _EncodeImage(0, ndf, cfg.GAN.LAYER_D_NUM)
        self.UNCOND_DNET = D_GET_LOGITS(ndf, nef, bcondition=False) if b_jcu else None
        self.COND_DNET = D_GET_LOGITS(ndf, nef, bcondition=True)
        self.out_channels = ndf * 8
        self.nhwc_features = True

    def forward(self, x_var):
        f = self.img_code(ops.to_nhwc(x_var))
        return NHWCFeature(f, self.out_channels) if self.nhwc_features else ops.to_nchw(f, self.out_channels)


class PAT_D_NET64(_PatD):
    """ref: model.py:1053-1068."""


class PAT_D_NET128(_PatD):
    """ref: model.py:1072-1087."""


class PAT_D_NET256(_PatD):
    """ref: model.py:1091-1106."""


# --------------------------------------------------------------------------------------------------
# shape discriminators (ref: model.py:1111-1179): image || shape-code(seg map) -> conv encoder; UNCOND head only
# --------------------------------------------------------------------------------------------------
class _ShpD(_Base):
    def __init__(self, num_classes):
        super().__init__()
        ndf, nef = cfg.GAN.DF_DIM, cfg.TEXT.EMBEDDING_DIM
        ngf = cfg.GAN.GF_DIM // 4
        self.img_code = _EncodeImage(ngf, ndf, cfg.GAN.LAYER_D_NUM)
        self.shp_code = _Slots(_1=Conv2dP(num_classes, ngf, 3, 1, 1, bias=True, mode=PAD_REFLECT))
        self.UNCOND_DNET = D_GET_LOGITS(ndf, nef, bcondition=False)
        self.ngf = ngf
        self.out_channels = ndf * 8
        self.nhwc_features = True

    def forward(self, x_var, s_var):
        new_s = ops.instance_norm_act(self.shp_code[1](ops.to_nhwc(s_var)), NA_LRELU)
        x_s = ops.cat_channels([ops.to_nhwc(x_var), new_s], [x_var.shape[1], self.ngf])
        f = self.img_code(x_s)
        return NHWCFeature(f, self.out_channels) if self.nhwc_features else ops.to_nchw(f, self.out_channels)


class SHP_D_NET64(_ShpD):
    """ref: model.py:1111-1132."""


class SHP_D_NET128(_ShpD):
    """ref: model.py:1135-1156."""


class SHP_D_NET256(_ShpD):
    """ref: model.py:1159-1179."""


# --------------------------------------------------------------------------------------------------
# object discriminators (ref: model.py:1184-1312): 512x512 bilinear front end, shape code, conv encoder,
# RoIAlignAvg over the 10 box slots of every image, roi code.  forward() returns (B, 10, 384, 4, 4) like the reference;
# the logit heads are D_GET_LOGITS(ndf // 2, nef) applied by objD_loss (loss glue: SURVEY 8f "next").
# --------------------------------------------------------------------------------------------------
class _ObjD(_Base):
    n_layer = 3

    def __init__(self, num_classes, b_jcu=True):
        super().__init__()
        ndf = cfg.GAN.DF_DIM
        nef = cfg.TEXT.GLOVE_EMBEDDING_DIM + cfg.GAN.GF_DIM
        ngf = cfg.GAN.GF_DIM // 4
        self.roi_size = cfg.ROI.ROI_BASE_SIZE
        self.im_scales = np.array([1])
        n_layer = self.n_layer
        self.img_code = _EncodeImage(ngf, ndf, n_layer)
        self.shp_code = _Slots(_1=Conv2dP(num_classes, ngf, 3, 1, 1, bias=True, mode=PAD_REFLECT))
        self.feat_dim = ndf * min(2 ** (n_layer - 1), 8)
        self.roi_code = _Slots(_0=Conv2dP(self.feat_dim, ndf * 4, 4, 1, 1, bias=True, act=ACT_LRELU))
        self.RoIAlignAvg = RoIAlignAvg(self.roi_size, self.roi_size, 1.0 / 16.0)
        self.UNCOND_DNET = D_GET_LOGITS(ndf // 2, nef, bcondition=False) if b_jcu else None
        self.COND_DNET = D_GET_LOGITS(ndf // 2, nef, bcondition=True)
        self.ngf = ngf

    def shape_features(self, s_var, img_size=512):
        """The shape branch (ref: model.py:1217-1219: bilinear -> ReflPad + conv3x3 80->12 + bias -> InstanceNorm ->
        LeakyReLU) of a segmentation map, NHWC.  It depends on the map and this net's weights only, so a loss that
        runs the net on several images with the SAME map (objD_loss: real and fake) computes it once and passes it
        to ``forward`` (autograd sums both uses' gradients): same values, one 80-channel 512^2 pass instead of two."""
        s = ops.cached_const(s_var, ("bilinear_nhwc", img_size),
                             lambda: ops.bilinear(ops.to_nhwc(s_var), img_size, img_size))   # same map for both object Ds
        return ops.instance_norm_act(self.shp_code[1](s), NA_LRELU)

    def forward(self, x_var, s_var, fm_rois, num_rois, img_size=512, shape_features=None):
        # (x, y, w, h) -> (x1, y1, x2, y2) on the host, on a COPY (the reference mutates a CPU caller's tensor in place,
        # ref: model.py:1213-1214; on CUDA it works on a copy too)
        fm = fm_rois.detach().cpu().numpy().astype(np.float64, copy=True)
        fm[:, :, [2, 3]] = fm[:, :, [0, 1]] + fm[:, :, [2, 3]]
        b = fm.shape[0]
        x = ops.bilinear(ops.to_nhwc(x_var), img_size, img_size)
        new_s = shape_features if shape_features is not None else self.shape_features(s_var, img_size)
        x_s = ops.cat_channels([x, new_s], [x_var.shape[1], self.ngf])
        code = self.img_code(x_s)                                           # NHWC (B, S/2^n, S/2^n, feat_dim)
        rois = _get_rois_blob(fm.reshape(b * fm.shape[1], fm.shape[2])[:, :4], np.array([1] * b * cfg.ROI.BOXES_NUM))
        rois_t = ops.h2d(rois, x_var.device)
        # the feature map is channels-last already: the channels-last RoIAlignAvg kernel (same values as the
        # reference-ABI NCHW op behind self.RoIAlignAvg) feeds roi_code without any layout round trip
        pooled = ops.roi_align_avg_nhwc(code, rois_t, self.RoIAlignAvg.aligned_height, self.RoIAlignAvg.aligned_width,
                                        self.RoIAlignAvg.spatial_scale)     # (B*10, 5, 5, C)
        pooled = self.roi_code[0](pooled)                                    # conv k4 s1 p1 + bias + LReLU
        out = ops.to_nchw(pooled, pooled.shape[3])
        return out.view(b, cfg.ROI.BOXES_NUM, out.shape[1], out.shape[2], out.shape[3])


class OBJ_SS_D_NET(_ObjD):
    """ref: model.py:1184-1246 (small-scale objects: 3 encoder layers, 64x64 feature map)."""
    n_layer = 3


class OBJ_LS_D_NET(_ObjD):
    """ref: model.py:1250-1312 (large-scale objects: 4 encoder layers, 32x32 feature map)."""
    n_layer = 4


# --------------------------------------------------------------------------------------------------
# ROIAlign modules (ref: models/roi_align/modules/roi_align.py) and the rois blob helper
# --------------------------------------------------------------------------------------------------
class RoIAlign(nn.Module):
    def __init__(self, aligned_height, aligned_width, spatial_scale):
        super().__init__()
        self.aligned_width, self.aligned_height = int(aligned_width), int(aligned_height)
        self.spatial_scale = float(spatial_scale)

    def forward(self, features, rois):
        return ops.roi_align(features, rois, self.aligned_height, self.aligned_width, self.spatial_scale)


class RoIAlignAvg(nn.Module):
    """ref: modules/roi_align.py:18-29 -- fused align (AH+1, AW+1) + avg_pool2d(2, 1) kernel."""

    def __init__(self, aligned_height, aligned_width, spatial_scale):
        super().__init__()
        self.aligned_width, self.aligned_height = int(aligned_width), int(aligned_height)
        self.spatial_scale = float(spatial_scale)

    def forward(self, features, rois):
        return ops.roi_align_avg(features, rois, self.aligned_height, self.aligned_width, self.spatial_scale)


def _get_rois_blob(im_rois, im_scale_factors):
    """ref: miscc/utils.py:365-399 (host numpy, float64 -> float32 [level, x1, y1, x2, y2])."""
    im_rois = np.asarray(im_rois, dtype=np.float64)
    n = cfg.ROI.BOXES_NUM
    levels = np.repeat(np.arange(im_rois.shape[0] // n), n).reshape(-1, 1)
    rois = im_rois * np.asarray(im_scale_factors, dtype=np.float64)[levels]
    return np.hstack((levels.astype(np.float64), rois)).astype(np.float32, copy=False)


# --------------------------------------------------------------------------------------------------
# DAMSM image encoder (ref: model.py:182-287): torchvision's Inception-v3 trunk from Conv2d_1a_3x3 to Mixed_7c,
# emb_features (1x1, 768 -> nef) on the Mixed_6e map and emb_cnn_code (Linear 2048 -> nef) on the 8x8 average.
# --------------------------------------------------------------------------------------------------
class _ConvWeight(nn.Module):
    """nn.Conv2d(bias=False) parameter holder (key ``weight``)."""

    def __init__(self, cin, cout, kh, kw):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, cin, kh, kw))
        nn.init.normal_(self.weight.data, 0.0, (1.0 / (cin * kh * kw)) ** 0.5)


class _BN(nn.Module):
    """nn.BatchNorm2d(eps=0.001) parameters and buffers (used in eval mode only)."""

    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))
        self.register_buffer("running_mean", torch.zeros(c))
        self.register_buffer("running_var", torch.ones(c))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))


class BasicConv2d(nn.Module):
    """torchvision's BasicConv2d: conv (no bias) -> BatchNorm2d(eps=0.001) -> ReLU; keys ``conv.weight``, ``bn.*``."""

    def __init__(self, cin, cout, k, stride=1, pad=(0, 0)):
        super().__init__()
        kh, kw = (k, k) if isinstance(k, int) else k
        self.conv = _ConvWeight(cin, cout, kh, kw)
        self.bn = _BN(cout)
        self.kh, self.kw, self.stride, self.pad = kh, kw, stride, pad

    def bn_tensors(self):
        return (self.bn.weight, self.bn.bias, self.bn.running_mean, self.bn.running_var)


# Inception-v3 blocks (torchvision.models.inception): per block kind, its BasicConv2d children as
# (name, cin, cout, kernel, stride, padding) with "IN" the block's input width and "C7" the InceptionC width.
_INCEPTION_CONVS = {
    "A": [("branch1x1", "IN", 64, 1, 1, 0), ("branch5x5_1", "IN", 48, 1, 1, 0), ("branch5x5_2", 48, 64, 5, 1, 2),
          ("branch3x3dbl_1", "IN", 64, 1, 1, 0), ("branch3x3dbl_2", 64, 96, 3, 1, 1),
          ("branch3x3dbl_3", 96, 96, 3, 1, 1), ("branch_pool", "IN", "PF", 1, 1, 0)],
    "B": [("branch3x3", "IN", 384, 3, 2, 0), ("branch3x3dbl_1", "IN", 64, 1, 1, 0), ("branch3x3dbl_2", 64, 96, 3, 1, 1),
          ("branch3x3dbl_3", 96, 96, 3, 2, 0)],
    "C": [("branch1x1", "IN", 192, 1, 1, 0), ("branch7x7_1", "IN", "C7", 1, 1, 0),
          ("branch7x7_2", "C7", "C7", (1, 7), 1, (0, 3)), ("branch7x7_3", "C7", 192, (7, 1), 1, (3, 0)),
          ("branch7x7dbl_1", "IN", "C7", 1, 1, 0), ("branch7x7dbl_2", "C7", "C7", (7, 1), 1, (3, 0)),
          ("branch7x7dbl_3", "C7", "C7", (1, 7), 1, (0, 3)), ("branch7x7dbl_4", "C7", "C7", (7, 1), 1, (3, 0)),
          ("branch7x7dbl_5", "C7", 192, (1, 7), 1, (0, 3)), ("branch_pool", "IN", 192, 1, 1, 0)],
    "D": [("branch3x3_1", "IN", 192, 1, 1, 0), ("branch3x3_2", 192, 320, 3, 2, 0),
          ("branch7x7x3_1", "IN", 192, 1, 1, 0), ("branch7x7x3_2", 192, 192, (1, 7), 1, (0, 3)),
          ("branch7x7x3_3", 192, 192, (7, 1), 1, (3, 0)), ("branch7x7x3_4", 192, 192, 3, 2, 0)],
    "E": [("branch1x1", "IN", 320, 1, 1, 0), ("branch3x3_1", "IN", 384, 1, 1, 0),
          ("branch3x3_2a", 384, 384, (1, 3), 1, (0, 1)), ("branch3x3_2b", 384, 384, (3, 1), 1, (1, 0)),
          ("branch3x3dbl_1", "IN", 448, 1, 1, 0), ("branch3x3dbl_2", 448, 384, 3, 1, 1),
          ("branch3x3dbl_3a", 384, 384, (1, 3), 1, (0, 1)), ("branch3x3dbl_3b", 384, 384, (3, 1), 1, (1, 0)),
          ("branch_pool", "IN", 192, 1, 1, 0)],
}
# (name, kind, input width, pool_features or c7)
_INCEPTION_BLOCKS = [("Mixed_5b", "A", 192, 32), ("Mixed_5c", "A", 256, 64), ("Mixed_5d", "A", 288, 64),
                     ("Mixed_6a", "B", 288, 0), ("Mixed_6b", "C", 768, 128), ("Mixed_6c", "C", 768, 160),
                     ("Mixed_6d", "C", 768, 160), ("Mixed_6e", "C", 768, 192), ("Mixed_7a", "D", 768, 0),
                     ("Mixed_7b", "E", 1280, 0), ("Mixed_7c", "E", 2048, 0)]
_STEM = [("Conv2d_1a_3x3", 3, 32, 3, 2, 0), ("Conv2d_2a_3x3", 32, 32, 3, 1, 0), ("Conv2d_2b_3x3", 32, 64, 3, 1, 1),
         ("Conv2d_3b_1x1", 64, 80, 1, 1, 0), ("Conv2d_4a_3x3", 80, 192, 3, 1, 0)]


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


class _InceptionBlock(nn.Module):
    def __init__(self, kind, cin, param):
        super().__init__()
        self.kind = kind
        sub = {"IN": cin, "PF": param, "C7": param}
        for name, ci, co, k, s, p in _INCEPTION_CONVS[kind]:
            self.add_module(name, BasicConv2d(sub.get(ci, ci), sub.get(co, co), _pair(k), s, _pair(p)))


def _enc_layer(convs, relu=True):
    c0 = convs[0]
    return ops.EncConv([c.conv.weight for c in convs], [c.bn_tensors() for c in convs], c0.kh, c0.kw, c0.stride,
                       c0.pad[0], c0.pad[1], eps=1e-3, relu=relu)


def _block_steps(blk, name, src, dst, chans):
    """Program steps of one Inception block: sibling 1x1 convolutions run as one GEMM (their weights concatenated
    along N); final branch outputs go into their channel slice of the block output."""
    s, L = [], lambda *n: _enc_layer([getattr(blk, m) for m in n])
    t = lambda x: f"{name}.{x}"

    def fused(names, outs):
        """siblings -> fused buffer, then each part to outs[i] = (buffer, channel offset)"""
        layer = L(*names)
        chans[t("fused")] = layer.cout
        s.append(("conv", layer, src, t("fused"), 0))
        off = 0
        for n, (d, doff) in zip(names, outs):
            co = getattr(blk, n).conv.weight.shape[0]
            if d != dst:
                chans[d] = co
            s.append(("copy", t("fused"), off, d, doff, co))
            off += co

    def conv(n, a, b, off=0, width=None):
        layer = L(n)
        if b != dst:
            chans[b] = layer.cout
        s.append(("conv", layer, a, b, off))
        return layer.cout

    def pool_branch(off):
        s.append(("avgpool", src, t("pool")))
        conv("branch_pool", t("pool"), dst, off)

    if blk.kind == "A":
        fused(["branch1x1", "branch5x5_1", "branch3x3dbl_1"], [(dst, 0), (t("b5"), 0), (t("d1"), 0)])
        conv("branch5x5_2", t("b5"), dst, 64)
        conv("branch3x3dbl_2", t("d1"), t("d2"))
        conv("branch3x3dbl_3", t("d2"), dst, 128)
        pool_branch(224)
        chans[dst] = 224 + blk.branch_pool.conv.weight.shape[0]
    elif blk.kind == "B":
        conv("branch3x3", src, dst, 0)
        conv("branch3x3dbl_1", src, t("d1"))
        conv("branch3x3dbl_2", t("d1"), t("d2"))
        conv("branch3x3dbl_3", t("d2"), dst, 384)
        s.append(("maxpool", src, dst, 480))
        chans[dst] = 480 + blk.branch3x3dbl_1.conv.weight.shape[1]
    elif blk.kind == "C":
        fused(["branch1x1", "branch7x7_1", "branch7x7dbl_1"], [(dst, 0), (t("a1"), 0), (t("d1"), 0)])
        conv("branch7x7_2", t("a1"), t("a2"))
        conv("branch7x7_3", t("a2"), dst, 192)
        conv("branch7x7dbl_2", t("d1"), t("d2"))
        conv("branch7x7dbl_3", t("d2"), t("d3"))
        conv("branch7x7dbl_4", t("d3"), t("d4"))
        conv("branch7x7dbl_5", t("d4"), dst, 384)
        pool_branch(576)
        chans[dst] = 768
    elif blk.kind == "D":
        fused(["branch3x3_1", "branch7x7x3_1"], [(t("a1"), 0), (t("b1"), 0)])
        conv("branch3x3_2", t("a1"), dst, 0)
        conv("branch7x7x3_2", t("b1"), t("b2"))
        conv("branch7x7x3_3", t("b2"), t("b3"))
        conv("branch7x7x3_4", t("b3"), dst, 320)
        s.append(("maxpool", src, dst, 512))
        chans[dst] = 512 + blk.branch3x3_1.conv.weight.shape[1]
    else:  # E
        fused(["branch1x1", "branch3x3_1", "branch3x3dbl_1"], [(dst, 0), (t("a1"), 0), (t("d1"), 0)])
        conv("branch3x3_2a", t("a1"), dst, 320)
        conv("branch3x3_2b", t("a1"), dst, 704)
        conv("branch3x3dbl_2", t("d1"), t("d2"))
        conv("branch3x3dbl_3a", t("d2"), dst, 1088)
        conv("branch3x3dbl_3b", t("d2"), dst, 1472)
        pool_branch(1856)
        chans[dst] = 2048
    return s


# stage outputs of the trunk: the two stem max-pools, then the blocks
_STAGES = ("stem2p", "stem4p") + tuple(b[0] for b in _INCEPTION_BLOCKS)


def _trunk_program(get, input_step, last, outputs, after=None):
    """torchvision's Inception-v3 trunk as an ops.InceptionProgram: ``input_step`` writes "x299" from "x", then the
    stem and the blocks run up to the stage ``last`` (a _STAGES name; "stem2p" / "stem4p" are the outputs of the
    first / second max-pool, the others the block outputs).  ``get(name)``: the BasicConv2d or _InceptionBlock of
    that torchvision name.  ``after``: {stage: (step, channels)} -- one more step that reads the stage's output
    (its destination has that many channels).  ``outputs``: the buffers the program returns; "pooled" adds the
    global average of the last stage."""
    if last not in _STAGES:
        raise ValueError(f"the trunk has no stage {last!r}; stages: {_STAGES}")
    after = after or {}
    steps, chans = [input_step], {}
    src = "x299"

    def staged(name):
        if name in after:
            step, c = after[name]
            chans[step[3]] = c
            steps.append(step)
        return name == last

    for i, (name, ci, co, k, s, p) in enumerate(_STEM):
        dst = f"stem{i}"
        chans[dst] = co
        steps.append(("conv", _enc_layer([get(name)]), src, dst, 0))
        src = dst
        if name in ("Conv2d_2b_3x3", "Conv2d_4a_3x3"):     # max_pool2d(3, 2) after these two
            chans[dst + "p"] = co
            steps.append(("maxpool", src, dst + "p", 0))
            src = dst + "p"
            if staged(src):
                break
    else:
        for name, kind, cin, param in _INCEPTION_BLOCKS:
            steps += _block_steps(get(name), name, src, name, chans)
            src = name
            if staged(name):
                break
    if "pooled" in outputs:
        steps.append(("gap", src, "pooled"))
    return ops.InceptionProgram(steps, chans, tuple(outputs))


class _FrozenInception(_Base):
    """Shared behaviour of the Inception-v3 networks: frozen and eval-only, a program rebuilt after .to() (the
    BatchNorm fold then reads the new buffers; loads are caught by the fold's version check), and state_dict loads
    that accept the ``module.`` prefix and snapshots without ``num_batches_tracked``."""
    _TRAIN_HINT = ""

    def _apply(self, fn, *a, **k):
        # .to() / .cuda() replace the BatchNorm buffers with new tensors: the program must fold from the new ones
        self._prog = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, strict=True, **kw):
        """Also takes keys with the ``module.`` prefix nn.DataParallel adds, and snapshots without the
        ``num_batches_tracked`` buffers (torch <= 0.4.0 did not write them)."""
        sd = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in state_dict.items()}
        for k, v in self.state_dict().items():
            if k.endswith(".num_batches_tracked") and k not in sd:
                sd[k] = v.clone()
        return super().load_state_dict(sd, strict=strict, **kw)

    def _check(self):
        name = type(self).__name__
        if self.training:
            raise RuntimeError(f"{name} runs in eval mode only (BatchNorm uses the running statistics); call "
                               f".eval(){self._TRAIN_HINT}")
        for n, p in self.named_parameters():
            if p.requires_grad:
                raise RuntimeError(f"{name} is frozen and computes no weight gradient, but {n} requires grad; "
                                   "call .requires_grad_(False)")


class CNN_ENCODER(_FrozenInception):
    """The DAMSM image encoder (ref: model.py:182-287) with the reference's state_dict keys and shapes.  It is frozen
    and eval-only, as the reference uses it (trainer.py:75-89, evaluator.py:97-105): the forward computes the input
    gradient (when the input requires grad) and never a weight gradient.  Construction reads no file; the trunk's
    weights start as fan-in-scaled normal draws until a snapshot is loaded.

    forward(x): x (B, 3, H, W) NCHW in [-1, 1] -> (features (B, nef, 17, 17), cnn_code (B, nef)).
    forward_nhwc(x): x (B, H, W, 8) NHWC with the channel pad lanes zero, same outputs."""
    _TRAIN_HINT = " -- training the image encoder (DAMSM pretraining) is not supported"

    def __init__(self, nef=256):
        super().__init__()
        self.nef = nef
        for name, ci, co, k, s, p in _STEM:
            self.add_module(name, BasicConv2d(ci, co, k, s, _pair(p)))
        for name, kind, cin, param in _INCEPTION_BLOCKS:
            self.add_module(name, _InceptionBlock(kind, cin, param))
        self.emb_features = _ConvWeight(768, nef, 1, 1)
        self.emb_cnn_code = LinearP(2048, nef)
        # ref: model.py:231-234 init_trainable_weights
        self.emb_features.weight.data.uniform_(-0.1, 0.1)
        self.emb_cnn_code.weight.data.uniform_(-0.1, 0.1)
        nn.init.uniform_(self.emb_cnn_code.bias.data, -(1 / 2048) ** 0.5, (1 / 2048) ** 0.5)
        self.requires_grad_(False)
        self.eval()
        self._prog = None

    @classmethod
    def from_snapshot(cls, path, device="cuda", nef=256):
        """The reference's ``image_encoder100.pth`` (keys with or without ``module.``)."""
        enc = cls(nef).to(device)
        enc.load_state_dict(torch.load(path, map_location="cpu"))
        return enc

    def program(self):
        """The forward as an ops.InceptionProgram (built once; it holds the parameters, not copies)."""
        if self._prog is None:
            emb = ("conv", ops.EncConv([self.emb_features.weight], None, 1, 1, relu=False), "Mixed_6e", "features", 0)
            self._prog = _trunk_program(lambda n: getattr(self, n), ("interp", "x", "x299", 299), "Mixed_7c",
                                        ("features", "pooled"), {"Mixed_6e": (emb, self.nef)})
        return self._prog

    def forward_nhwc(self, x):
        self._check()
        feat, pooled = ops.inception_trunk(x, self.program())
        cnn_code = self.emb_cnn_code(pooled)
        return ops.to_nchw(feat, self.nef), cnn_code

    def forward(self, x):
        assert x.dim() == 4 and x.shape[1] == 3, "CNN_ENCODER takes (B, 3, H, W) images"
        self._check()
        return self.forward_nhwc(ops.to_nhwc(x))


# --------------------------------------------------------------------------------------------------
# Scoring networks (ref: model.py:290-451): the ImageNet Inception-v3 for the Inception score and for the FID
# activations.  Same trunk as CNN_ENCODER, another input transform, and forward only.
# --------------------------------------------------------------------------------------------------
IS_INPUT, FID_INPUT = 0, 1      # og_inception_input modes
# torchvision's Inception3 stem / block names in INCEPTION_V3_FID's blocks.<i>.<j> layout
_FID_BLOCKS = (("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3"), ("Conv2d_3b_1x1", "Conv2d_4a_3x3"),
               ("Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"),
               ("Mixed_7a", "Mixed_7b", "Mixed_7c"))
_FID_LAST = ("stem2p", "stem4p", "Mixed_6e", "Mixed_7c")      # the trunk stage that ends each block
_FID_OUT = ("stem2p", "stem4p", "Mixed_6e", "pooled")


def _imagenet_state_dict(src):
    """torchvision's ``inception_v3_google-1a9a5a14.pth`` (keys as Inception3's, also with ``module.``), from its path
    or as already loaded."""
    sd = src if isinstance(src, dict) else torch.load(src, map_location="cpu")
    return {(k[len("module."):] if k.startswith("module.") else k): v for k, v in sd.items()}


class _InceptionAux(nn.Module):
    """torchvision's InceptionAux parameters (held and loaded; the eval forward never runs it)."""

    def __init__(self):
        super().__init__()
        self.conv0 = BasicConv2d(768, 128, 1)
        self.conv1 = BasicConv2d(128, 768, 5)
        self.fc = LinearP(768, 1000)


class _Inception3(nn.Module):
    """torchvision's Inception3(aux_logits=True, num_classes=1000) state_dict layout."""

    def __init__(self):
        super().__init__()
        for name, ci, co, k, s, p in _STEM:
            self.add_module(name, BasicConv2d(ci, co, k, s, _pair(p)))
        for name, kind, cin, param in _INCEPTION_BLOCKS:
            self.add_module(name, _InceptionBlock(kind, cin, param))
            if name == "Mixed_6e":
                self.AuxLogits = _InceptionAux()
        self.fc = LinearP(2048, 1000)


class INCEPTION_V3(_FrozenInception):
    """The Inception-score network (ref: model.py:290-315) with the reference's state_dict keys (``model.`` plus
    torchvision's Inception3 keys, AuxLogits included).  Frozen, eval-only, forward-only: the output carries no
    gradient.  Each rank of a data-parallel run scores its own images; predictions are not gathered.

    forward(x): x (B, 3, H, W) in [-1, 1] -> (B, 1000) class probabilities.  The input goes through x * 0.5 + 0.5,
    the ImageNet normalisation and the align_corners=True resize to 299 (og_inception_input), the trunk to Mixed_7c,
    the 8x8 average, ``fc`` and a row softmax (og_softmax_rows)."""

    def __init__(self):
        super().__init__()
        self.model = _Inception3()
        self.requires_grad_(False)
        self.eval()
        self._prog = None

    @classmethod
    def from_imagenet(cls, path, device="cuda"):
        """torchvision's ImageNet file ``inception_v3_google-1a9a5a14.pth`` (its path, or its state_dict already
        loaded), as the reference loads it."""
        net = cls().to(device)
        net.load_state_dict({"model." + k: v for k, v in _imagenet_state_dict(path).items()})
        return net

    def program(self):
        if self._prog is None:
            self._prog = _trunk_program(lambda n: getattr(self.model, n), ("input", "x", "x299", 299, IS_INPUT),
                                        "Mixed_7c", ("pooled",))
        return self._prog

    def forward(self, x):
        assert x.dim() == 4 and x.shape[1] == 3, "INCEPTION_V3 takes (B, 3, H, W) images"
        self._check()
        with torch.no_grad():
            pooled = self.program().forward(x.detach().float().contiguous())["pooled"]
            return ops.softmax_rows(self.model.fc(pooled))


class INCEPTION_V3_FID(_FrozenInception):
    """The FID network (ref: model.py:318-451) with the reference's ``blocks.<i>.<j>`` state_dict keys, holding only
    the blocks up to the last one requested.  Frozen, eval-only, forward-only.

    Blocks: 0 ends at the first max-pool (64 channels), 1 at the second (192), 2 at Mixed_6e (768), 3 at the Mixed_7c
    average (2048).  The input goes through the half-pixel resize to 299, then x * 0.5 + 0.5 and the reference's
    x * (std / 0.5) + (mean - 0.5) / 0.5 (og_inception_input); the trunk stops at the last requested block.

    forward(x): x (B, 3, H, W) in [-1, 1] -> the list of the requested blocks' maps (B, C, h, w), by block index.
    activations(x): the first requested block's map averaged over its pixels, (B, C) -- the reference's
    get_activations (utils.py:587-641)."""
    DEFAULT_BLOCK_INDEX = 3
    BLOCK_INDEX_BY_DIM = {64: 0, 192: 1, 768: 2, 2048: 3}

    def __init__(self, output_blocks=(DEFAULT_BLOCK_INDEX,)):
        super().__init__()
        self.output_blocks = sorted(output_blocks)
        if not self.output_blocks or self.output_blocks[0] < 0 or self.output_blocks[-1] > 3:
            raise ValueError(f"output_blocks must be block indices in 0..3, got {list(output_blocks)}")
        self.last_needed_block = self.output_blocks[-1]
        self.blocks = nn.ModuleList()
        for b in range(self.last_needed_block + 1):
            mods = nn.ModuleList()
            for name in _FID_BLOCKS[b]:
                kind = next((k for n, k, c, q in _INCEPTION_BLOCKS if n == name), None)
                if kind is None:
                    ci, co, k, s, p = next(r[1:] for r in _STEM if r[0] == name)
                    mods.append(BasicConv2d(ci, co, k, s, _pair(p)))
                else:
                    cin, param = next((c, q) for n, k, c, q in _INCEPTION_BLOCKS if n == name)
                    mods.append(_InceptionBlock(kind, cin, param))
            self.blocks.append(mods)
        self.requires_grad_(False)
        self.eval()
        self._prog = None

    @classmethod
    def from_imagenet(cls, path, device="cuda", output_blocks=(DEFAULT_BLOCK_INDEX,)):
        """torchvision's ImageNet file ``inception_v3_google-1a9a5a14.pth`` (its path, or its state_dict already
        loaded); only the needed blocks are read."""
        net = cls(output_blocks).to(device)
        net.load_state_dict(net.from_torchvision(_imagenet_state_dict(path)))
        return net

    def from_torchvision(self, sd):
        """This module's state_dict from an Inception3 one (torchvision keys)."""
        out = {}
        for b, names in enumerate(_FID_BLOCKS[:self.last_needed_block + 1]):
            for j, name in enumerate(names):
                for k, v in sd.items():
                    if k.startswith(name + "."):
                        out[f"blocks.{b}.{j}.{k[len(name) + 1:]}"] = v
        return out

    def _module(self, name):
        for b, names in enumerate(_FID_BLOCKS):
            if name in names:
                return self.blocks[b][names.index(name)]
        raise KeyError(name)

    def program(self):
        if self._prog is None:
            self._prog = _trunk_program(self._module, ("input", "x", "x299", 299, FID_INPUT),
                                        _FID_LAST[self.last_needed_block],
                                        tuple(_FID_OUT[b] for b in self.output_blocks))
        return self._prog

    def _outputs(self, x):
        assert x.dim() == 4 and x.shape[1] == 3, "INCEPTION_V3_FID takes (B, 3, H, W) images"
        self._check()
        bufs = self.program().forward(x.detach().float().contiguous())
        return [bufs[_FID_OUT[b]] for b in self.output_blocks]

    def forward(self, x):
        with torch.no_grad():
            return [y.view(y.shape[0], -1, 1, 1) if y.dim() == 2 else ops.to_nchw(y, y.shape[-1])
                    for y in self._outputs(x)]

    def activations(self, x):
        with torch.no_grad():
            y = self._outputs(x)[0]
            if y.dim() == 2:
                return y
            n, h, w, c = y.shape
            out = torch.empty((n, c), device=y.device, dtype=torch.float32)
            ops._call("og_global_avg_fwd", ops._p(y), n, h * w, c, ops._p(out))
            return out
