"""CPU restatement (torch.nn.functional on fp32 CPU tensors) of the shape-generation path of the reference's evaluator:
the box maps its loader builds from a layout, SHP_G_NET's forward over a state_dict, and form_hmaps.  Every function
cites the reference lines it restates (paths under image_generation/ of the original project).  The tests compare it
with the reference's own modules (tests/golden/reference/shp_g_net_*.npz, form_hmaps_gen.npz) and the CUDA path with it.
"""
import numpy as np
import torch
import torch.nn.functional as F

BOXES_NUM = 10          # ref: miscc/config.py:81
FM_SIZE = 16            # ref: miscc/config.py:83
R_NUM = 1               # ref: miscc/config.py:68
IN_EPS = 1e-5           # nn.InstanceNorm2d default
LRELU = 0.2


# ---------------------------------------------------------------------------------------------------------------------
# box maps (ref: miscc/load.py:625-641 rasterises, load.py:178-189 / 201-212 places them per slot and reverses)
# ---------------------------------------------------------------------------------------------------------------------
def _edge(v, size):
    """min(int(round(v)), size - 1): Python's round of a float is round-half-to-even (load.py:628-631)."""
    return min(int(round(float(v))), size - 1)


def box_mask(x, y, w, h, size):
    """One box rasterised like load.py:626-632: [y0:y1, x0:x1] = 1 with Python slice bounds (upper bound exclusive)."""
    m = np.zeros((size, size))
    m[_edge(y, size):_edge(y + h, size), _edge(x, size):_edge(x + w, size)] = 1
    return m


def bbox_maps(rois0, fm_rois, num_rois, rmax, num_classes, size=64, fsize=FM_SIZE, boxes=BOXES_NUM):
    """(bbox_maps_fwd (B, rmax, num_classes, size, size), bbox_maps_bwd (same), bbox_fmaps (B, rmax, fsize, fsize)) as
    float32 tensors from the box tables: rois0 / fm_rois (B, boxes, >=5) float64 rows (x, y, w, h, cls) at 64 / 32
    pixels, num_rois (B,).  The backward sequence reverses all ``boxes`` slots before the [:rmax] slice (load.py:188,
    testDataset.py:148-150)."""
    rois0 = np.asarray(rois0, dtype=np.float64)
    fm_rois = np.asarray(fm_rois, dtype=np.float64)
    B = rois0.shape[0]
    fwd_all, bwd_all, fm_all = [], [], []
    for b in range(B):
        n = int(num_rois[b])
        fwd = np.zeros((boxes, num_classes, size, size))
        fmaps = np.zeros((boxes, fsize, fsize))
        for r in range(n):
            x, y, w, h = rois0[b, r, :4]
            fwd[r, int(rois0[b, r, 4])] = box_mask(x, y, w, h, size)                         # load.py:186-187
            fx, fy, fw, fh = fm_rois[b, r, :4]                                               # load.py:637-641 (32 -> 16)
            fmaps[r][_edge(fy / 2.0, fsize):_edge(fy / 2.0 + fh / 2.0, fsize),
                     _edge(fx / 2.0, fsize):_edge(fx / 2.0 + fw / 2.0, fsize)] = 1
        bwd = fwd[::-1].copy()                                                               # load.py:188
        fwd_all.append(fwd[:rmax])
        bwd_all.append(bwd[:rmax])
        fm_all.append(fmaps[:rmax])
    f = lambda a: torch.from_numpy(np.stack(a)).float()
    return f(fwd_all), f(bwd_all), f(fm_all)


# ---------------------------------------------------------------------------------------------------------------------
# SHP_G_NET (ref: model.py:798-985)
# ---------------------------------------------------------------------------------------------------------------------
def _in(x):
    return F.instance_norm(x, eps=IN_EPS)


def _glu(x):
    nc = x.size(1) // 2                                                                      # model.py:19-27
    return x[:, :nc] * torch.sigmoid(x[:, nc:])


def down_block(sd, p, x):
    """downBlock_3x3 (model.py:800-806)."""
    return F.leaky_relu(_in(F.conv2d(x, sd[p + ".0.weight"], stride=2, padding=1)), LRELU)


def clstm_cell(sd, p, x, state):
    """CLSTMCell.forward (model.py:828-863); state None = zero state."""
    hidden = sd[p + ".Gates.weight"].shape[0] // 4
    if state is None:
        z = torch.zeros(x.shape[0], hidden, x.shape[2], x.shape[3])
        state = (z, z)
    prev_hidden, prev_cell = state
    gates = F.conv2d(torch.cat((x, prev_hidden), 1), sd[p + ".Gates.weight"], sd[p + ".Gates.bias"], padding=1)
    in_gate, remember_gate, out_gate, cell_gate = gates.chunk(4, 1)
    in_gate, remember_gate, out_gate = torch.sigmoid(in_gate), torch.sigmoid(remember_gate), torch.sigmoid(out_gate)
    cell_gate = torch.tanh(cell_gate)
    cell = (remember_gate * prev_cell) + (in_gate * cell_gate)
    return out_gate * torch.tanh(cell), cell


def lstm_gates(gates, prev_cell):
    """The cell's pointwise part on precomputed gates (what og_clstm_cell does after its gate sum)."""
    in_gate, remember_gate, out_gate, cell_gate = gates.chunk(4, 1)
    in_gate, remember_gate, out_gate = torch.sigmoid(in_gate), torch.sigmoid(remember_gate), torch.sigmoid(out_gate)
    cell = (remember_gate * prev_cell) + (in_gate * torch.tanh(cell_gate))
    return out_gate * torch.tanh(cell), cell


def res_block(sd, p, x):
    """ResBlock(norm=nn.InstanceNorm2d) (model.py:866-882)."""
    y = _glu(_in(F.conv2d(x, sd[p + ".block.0.weight"], padding=1)))
    y = _glu(_in(F.conv2d(y, sd[p + ".block.3.weight"], padding=1)))
    return F.conv2d(y, sd[p + ".block.6.weight"], padding=1) + x


def up_block(sd, p, x):
    """upBlock(norm=nn.InstanceNorm2d) (model.py:43-49)."""
    x = F.interpolate(x, scale_factor=2, mode="nearest")
    return _glu(_in(F.conv2d(x, sd[p + ".1.weight"], padding=1)))


def shp_g_net_forward(sd, z_code, bbox_maps_fwd, bbox_maps_bwd, bbox_fmaps, fm_size=FM_SIZE, r_num=R_NUM):
    """SHP_G_NET.forward (model.py:920-985): z_code (B, R, 4*nbf) -> (B, R, 1, S, S)."""
    nbf = sd["img_net.img.0.weight"].shape[1]
    b, r = z_code.size(0), z_code.size(1)
    z = z_code.unsqueeze(3).repeat(1, 1, 1, fm_size ** 2).view(b, r, -1, fm_size, fm_size)      # 929-935
    s = bbox_maps_fwd.size(3)
    hf = down_block(sd, "downsample2", down_block(sd, "downsample1", bbox_maps_fwd.reshape(-1, nbf, s, s)))
    hf = hf.view(b, r, -1, fm_size, fm_size)                                                     # 938-942
    hb = down_block(sd, "downsample2", down_block(sd, "downsample1", bbox_maps_bwd.reshape(-1, nbf, s, s)))
    hb = hb.view(b, r, -1, fm_size, fm_size)                                                     # 944-947
    sf = sb = None
    fl, bl = [], []
    for t in range(r):                                                                           # 950-957
        sf = clstm_cell(sd, "fwd_convlstm", hf[:, t], sf)
        fl.append(sf[0].unsqueeze(1))
        sb = clstm_cell(sd, "bwd_convlstm", hb[:, t], sb)
        bl.append(sb[0].unsqueeze(1))
    h = torch.cat([torch.cat((fl[t], bl[r - t - 1], z[:, t:t + 1]), 2) for t in range(r)], 1)   # 960-963
    h = h.view(b * r, -1, fm_size, fm_size)
    h = _glu(_in(F.conv2d(h, sd["jointConv.0.weight"], padding=1)))                             # 967
    fm = bbox_fmaps.unsqueeze(2).repeat(1, 1, nbf * 4, 1, 1).view(b * r, -1, fm_size, fm_size)   # 970-972
    h = h * fm
    for i in range(r_num):                                                                       # 975
        h = res_block(sd, f"residual.{i}", h)
    h = up_block(sd, "upsample2", up_block(sd, "upsample1", h))                                 # 978-979
    out = torch.sigmoid(F.conv2d(h, sd["img_net.img.0.weight"]))                                 # 885-895
    return out.view(b, r, -1, s, s)


# ---------------------------------------------------------------------------------------------------------------------
# form_hmaps (ref: miscc/utils.py:524-584)
# ---------------------------------------------------------------------------------------------------------------------
def _renorm(m):
    lo, hi = torch.min(m), torch.max(m)
    if lo != hi:
        return (m - lo) / (hi - lo)
    if hi < 0.6:
        return m * 0
    return m


def form_hmaps(raw_masks, num_rois, roi_cls, hmap_size=(64, 128, 256), num_classes=80):
    """raw_masks (B, R, S, S), num_rois (B,), roi_cls (B, >=R) class ids -> (hmaps[3] (B, num_classes, s, s),
    bt_masks[3] (B, R, s, s), fm_bt_masks (B, R, s0/2, s0/2)).  Slots >= num_rois[b] keep their raw values."""
    b = raw_masks.size(0)
    top = hmap_size[-1]
    re = F.interpolate(raw_masks, size=(top, top), mode="bilinear", align_corners=True)        # 529-530
    hm = torch.zeros(b, num_classes, top, top)
    for i in range(b):
        cats = [int(c) for c in roi_cls[i, :int(num_rois[i])].tolist()]
        for count, c in enumerate(cats):                                                         # 542-558
            m = _renorm(re[i, count])
            re[i, count] = m
            hm[i, c] = torch.max(torch.cat((m.unsqueeze(0), hm[i, c].unsqueeze(0)), 0), 0)[0]
        for c in cats:                                                                           # 560-568
            hm[i, c] = _renorm(hm[i, c])
    rs = lambda x, s: F.interpolate(x, size=(s, s), mode="bilinear", align_corners=True)
    hmaps = [rs(hm, s) for s in hmap_size]                                                       # 570-579
    bt_masks = [rs(re, s) for s in hmap_size]
    return hmaps, bt_masks, rs(re, hmap_size[0] // 2)                                            # 581-582
