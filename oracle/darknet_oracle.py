"""ORACLE -- test infrastructure only.  CPU restatement (plain torch fp32 functional ops + numpy) of the
reference's hot path.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
import this; nothing under the product package does.

Every function cites the reference file:line (relative to /root/reference) whose algorithm it restates.  The
arithmetic itself lives in third-party PyTorch (requirements.txt:4 `torch>=1.5.1`; this image: 2.11.0+cu128):
nn.Conv2d / BatchNorm2d / LeakyReLU / Upsample / MaxPool2d call sites models.py:92-225, F.softplus/tanh
utils/layers.py:148, nn.BCEWithLogitsLoss utils/utils.py:376-377.

Pinned: tests/test_oracle_golden.py checks this file against tests/golden/*.npz, which oracle/gen_golden.py
produced by importing and running the reference itself (here, on CPU) on seeded inputs.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


# ------------------------------------------------------------------------------------------------------------------
# deterministic synthetic parameters, keyed by state_dict name (identical for the reference model and ours)
# ------------------------------------------------------------------------------------------------------------------
def synth_state_dict(ref_state, seed=0):
    """Fill a state_dict (name -> tensor, any framework-owned tensors) with reproducible values:
    conv weights ~ N(0, 1/fan_in), BN gamma ~ U(0.8, 1.2), beta ~ N(0, 0.1), running_mean ~ N(0, 0.1),
    running_var ~ U(0.8, 1.2), biases ~ N(0, 0.1)   (SURVEY.md section 8d).  Order-independent: every tensor has its
    own RandomState seeded from (seed, crc32(name))."""
    import zlib
    out = {}
    for name, t in ref_state.items():
        shape = tuple(t.shape)
        rs = np.random.RandomState((seed * 1000003 + zlib.crc32(name.encode())) % (2 ** 31))
        if name.endswith('num_batches_tracked'):
            out[name] = torch.zeros(shape, dtype=torch.long)
            continue
        if name.endswith('running_var') or (name.endswith('.weight') and 'BatchNorm2d' in name) or \
                name.endswith('gamma'):
            v = rs.uniform(0.8, 1.2, size=shape)
        elif name.endswith('.weight') and len(shape) >= 2:
            fan_in = int(np.prod(shape[1:]))
            v = rs.normal(0.0, 1.0 / math.sqrt(fan_in), size=shape)
        else:
            v = rs.normal(0.0, 0.1, size=shape)
        out[name] = torch.from_numpy(np.asarray(v, dtype=np.float32)).reshape(shape)
    return out


def synth_images(batch, h, w, seed=0):
    """uint8 images -> float /256 (train.py:348; NB the reference divides by 256 in train and test)."""
    rs = np.random.RandomState(seed)
    img = rs.randint(0, 256, size=(batch, 3, h, w)).astype(np.uint8)
    return torch.from_numpy(img).float() / 256.0


def synth_targets(batch, per_image=8, nc=80, seed=1):
    """[nT,6] rows (image, class, x, y, w, h), x,y in [0.05,0.95), w,h log-uniform in [0.02,0.6]."""
    rs = np.random.RandomState(seed)
    n = batch * per_image
    img = np.repeat(np.arange(batch), per_image).astype(np.float32)
    cls = rs.randint(0, nc, size=n).astype(np.float32)
    xy = rs.uniform(0.05, 0.95, size=(n, 2)).astype(np.float32)
    wh = np.exp(rs.uniform(math.log(0.02), math.log(0.6), size=(n, 2))).astype(np.float32)
    return torch.from_numpy(np.concatenate([img[:, None], cls[:, None], xy, wh], 1))


# ------------------------------------------------------------------------------------------------------------------
# activations -- models.py:102-113, utils/layers.py:141-173
# ------------------------------------------------------------------------------------------------------------------
def activation(x, name, slope=0.1):
    if name == 'leaky':
        return F.leaky_relu(x, slope)          # models.py:103
    if name == 'mish':
        return x * F.softplus(x).tanh()        # utils/layers.py:146-148
    if name == 'relu6':
        return F.relu6(x)                      # utils/layers.py:151-156
    if name == 'h_swish':
        return x * (F.relu6(x + 3.0) / 6.0)    # utils/layers.py:159-164
    if name == 'relu':
        return F.relu(x)
    if name == 'swish':
        return x * torch.sigmoid(x)            # utils/layers.py:141-143
    return x                                    # 'linear'


def mish_backward(x, grad_output):
    """utils/layers.py:123-128 (MishImplementation.backward)."""
    sx = torch.sigmoid(x)
    fx = F.softplus(x).tanh()
    return grad_output * (fx + x * sx * (1 - fx * fx))


def fold_bn(w, conv_bias, gamma, beta, mean, var, eps):
    """utils/torch_utils.py:65-89 (fuse_conv_and_bn) -> (w_folded, bias_folded)."""
    scale = gamma / torch.sqrt(eps + var)
    wf = w * scale.view(-1, 1, 1, 1)
    b = conv_bias if conv_bias is not None else torch.zeros_like(mean)
    bf = scale * b + beta - gamma * mean / torch.sqrt(var + eps)
    return wf, bf


# ------------------------------------------------------------------------------------------------------------------
# YOLO layer -- models.py:350-437
# ------------------------------------------------------------------------------------------------------------------
def yolo_layer(p_nchw, anchors_px, stride, nc, training):
    """p_nchw [B, na*no, ny, nx] -> training: p [B,na,ny,nx,no]; eval: (io [B, na*ny*nx, no], p)."""
    anchors = torch.as_tensor(np.asarray(anchors_px), dtype=torch.float32)
    na, no = anchors.shape[0], nc + 5
    bs, _, ny, nx = p_nchw.shape
    p = p_nchw.view(bs, na, no, ny, nx).permute(0, 1, 3, 4, 2).contiguous()          # models.py:406
    if training:
        return p
    yv, xv = torch.meshgrid([torch.arange(ny), torch.arange(nx)], indexing='ij')    # models.py:373
    grid = torch.stack((xv, yv), 2).view(1, 1, ny, nx, 2).float()                  # models.py:374
    anchor_wh = (anchors / stride).view(1, na, 1, 1, 2)                            # models.py:362-363
    io = p.clone()
    io[..., :2] = torch.sigmoid(io[..., :2]) + grid                                # models.py:415
    io[..., 2:4] = torch.exp(io[..., 2:4]) * anchor_wh                             # models.py:416
    io[..., :4] *= stride                                                          # models.py:417
    torch.sigmoid_(io[..., 4:])                                                    # models.py:418
    return io.view(bs, -1, no), p                                                  # models.py:437


def yolo_strides(cfg_name, n_yolo):
    """models.py:312-315: [32,16,8], reversed when the cfg *path* contains panet|yolov4|cd53 and not yolov4-tiny."""
    stride = [32, 16, 8]
    if any(x in cfg_name for x in ['panet', 'yolov4', 'cd53']) and 'yolov4-tiny' not in cfg_name:
        stride = list(reversed(stride))
    return stride[:n_yolo]


# ------------------------------------------------------------------------------------------------------------------
# Darknet forward -- models.py:508-561 (forward_once), create_modules branches models.py:29-335
# ------------------------------------------------------------------------------------------------------------------
def darknet_forward(module_defs, state, x, cfg_name, training=False, emulate_fp16=False, bn_momentum=0.1,
                    maxabsscaler=False, return_layers=False):
    """module_defs: parsed cfg WITHOUT the [net] block; state: state_dict (reference key names).
    eval  -> (io_cat [B, rows, no], [p...])          training -> [p...]  (+ dict of updated running stats)
    emulate_fp16: weights (after BN fold) and every layer output are rounded to fp16, accumulation stays fp32 --
    the precision policy of the H100 engine (config C1), used to gate the CUDA path tightly."""
    outs = []
    yolo_out = []
    n_yolo = sum(1 for d in module_defs if d['type'] == 'yolo')
    strides = yolo_strides(cfg_name, n_yolo)
    yi = -1
    rnd = (lambda t: t.half().float()) if emulate_fp16 else (lambda t: t)
    new_stats = {}
    in_ch = [x.shape[1]]
    for i, d in enumerate(module_defs):
        t = d['type']
        pre = 'module_list.%d.' % i
        if t in ('convolutional', 'depthwise'):
            # depthwise (models.py:115-197): the same block with Conv2d(groups=Cin) registered as 'DepthWise2d'
            cname = 'Conv2d.' if t == 'convolutional' else 'DepthWise2d.'
            groups = x.shape[1] if t == 'depthwise' else 1
            k = int(d['size'])
            pad = (k - 1) // 2 if int(d['pad']) else 0                               # models.py:33, 119
            w = state[pre + cname + 'weight']
            b = state.get(pre + cname + 'bias')
            slope = 0.25 if maxabsscaler else 0.1
            head = (i + 1 < len(module_defs) and module_defs[i + 1]['type'] == 'yolo')
            if int(d['batch_normalize']) and not training:
                wf, bf = fold_bn(w, b, state[pre + 'BatchNorm2d.weight'], state[pre + 'BatchNorm2d.bias'],
                                 state[pre + 'BatchNorm2d.running_mean'], state[pre + 'BatchNorm2d.running_var'], 1e-5)
                if emulate_fp16 and i > 0:
                    wf = wf.half().float()
                y = F.conv2d(x, wf, bf, stride=int(d['stride']), padding=pad, groups=groups)
            elif int(d['batch_normalize']):
                wq = w.half().float() if (emulate_fp16 and i > 0) else w
                y = F.conv2d(x, wq, None, stride=int(d['stride']), padding=pad, groups=groups)
                g_, b_ = state[pre + 'BatchNorm2d.weight'], state[pre + 'BatchNorm2d.bias']
                rm = state[pre + 'BatchNorm2d.running_mean'].clone()
                rv = state[pre + 'BatchNorm2d.running_var'].clone()
                if emulate_fp16:
                    # engine policy: statistics from the fp32 accumulators, normalisation applied to the fp16-stored z
                    mean = y.mean(dim=(0, 2, 3))
                    var = y.var(dim=(0, 2, 3), unbiased=False)
                    n_ = y.numel() / y.shape[1]
                    with torch.no_grad():
                        rm.mul_(1 - bn_momentum).add_(bn_momentum * mean)
                        rv.mul_(1 - bn_momentum).add_(bn_momentum * var * n_ / max(n_ - 1, 1))
                    z16 = y.half().float()
                    y = (z16 - mean.view(1, -1, 1, 1)) / torch.sqrt(var.view(1, -1, 1, 1) + 1e-5) \
                        * g_.view(1, -1, 1, 1) + b_.view(1, -1, 1, 1)
                else:
                    y = F.batch_norm(y, rm, rv, g_, b_, True, bn_momentum, 1e-5)    # models.py:100
                new_stats[pre + 'BatchNorm2d.running_mean'] = rm
                new_stats[pre + 'BatchNorm2d.running_var'] = rv
            else:
                wq = w.half().float() if (emulate_fp16 and i > 0) else w
                y = F.conv2d(x, wq, b, stride=int(d['stride']), padding=pad, groups=groups)
            y = activation(y, d['activation'], slope)
            x = y if head else rnd(y)
        elif t == 'se':
            # squeeze-excite (utils/layers.py:176-192): x * hsigmoid(W2 relu(W1 avgpool(x))), both Linear without bias
            w1, w2 = state[pre + 'se.fc.0.weight'], state[pre + 'se.fc.2.weight']
            sq = x.mean(dim=(2, 3))
            ex = F.relu6(F.linear(F.relu(F.linear(sq, w1)), w2) + 3.0) / 6.0
            x = rnd(x * ex.view(x.shape[0], x.shape[1], 1, 1))
        elif t == 'maxpool':
            k, s = d['size'], d['stride']
            if k == 2 and s == 1:                                                   # models.py:211-213
                x = F.max_pool2d(F.pad(x, (0, 1, 0, 1)), k, s, (k - 1) // 2)
            else:
                x = F.max_pool2d(x, k, s, (k - 1) // 2)                            # models.py:210
        elif t == 'upsample':
            x = F.interpolate(x, scale_factor=d['stride'])                          # models.py:225 (nearest)
        elif t == 'route':                                                          # utils/layers.py:26-40
            layers = d['layers']
            if len(layers) > 1:
                x = torch.cat([outs[l] for l in layers], 1)
            elif 'groups' in d:
                x = x[:, (x.shape[1] // 2):]
            else:
                x = outs[layers[0]]
        elif t == 'shortcut':                                                       # utils/layers.py:43-72
            for l in d['from']:
                a = outs[l]
                nx_, na_ = x.shape[1], a.shape[1]
                if nx_ == na_:
                    x = x + a
                elif nx_ > na_:
                    x = x.clone()
                    x[:, :na_] = x[:, :na_] + a
                else:
                    x = x + a[:, :nx_]
            x = rnd(x)
        elif t == 'yolo':
            yi += 1
            anchors = np.asarray(d['anchors'])[d['mask']]                           # models.py:317
            yolo_out.append(yolo_layer(x, anchors, strides[yi], int(d['classes']), training))
        else:
            raise NotImplementedError(t)
        outs.append(x)
    if return_layers == 'both':
        return yolo_out, outs
    if return_layers:
        return outs
    if training:
        return yolo_out, new_stats
    io, p = zip(*yolo_out)
    return torch.cat(io, 1), list(p)                                                # models.py:553-554


# ------------------------------------------------------------------------------------------------------------------
# loss -- utils/utils.py:254-297 (bbox_iou), 325-330 (wh_iou), 368-432 (compute_loss), 725-779 (build_targets)
# ------------------------------------------------------------------------------------------------------------------
DEFAULT_HYP = {'giou': 3.54, 'cls': 37.4, 'cls_pw': 1.0, 'obj': 64.3, 'obj_pw': 1.0, 'iou_t': 0.20, 'fl_gamma': 0.0}
# train.py:25-31; train.py:87 scales hyp['cls'] *= nc / 80


def wh_iou(wh1, wh2):
    wh1 = wh1[:, None]
    wh2 = wh2[None]
    inter = torch.min(wh1, wh2).prod(2)
    return inter / (wh1.prod(2) + wh2.prod(2) - inter)                              # utils.py:325-330


def giou_xywh(box1_t, box2):
    """bbox_iou(box1.t(), box2, x1y1x2y2=False, GIoU=True): box1_t [4,n], box2 [n,4]  (utils.py:254-283)."""
    box2 = box2.t()
    b1_x1, b1_x2 = box1_t[0] - box1_t[2] / 2, box1_t[0] + box1_t[2] / 2
    b1_y1, b1_y2 = box1_t[1] - box1_t[3] / 2, box1_t[1] + box1_t[3] / 2
    b2_x1, b2_x2 = box2[0] - box2[2] / 2, box2[0] + box2[2] / 2
    b2_y1, b2_y2 = box2[1] - box2[3] / 2, box2[1] + box2[3] / 2
    inter = (torch.min(b1_x2, b2_x2) - torch.max(b1_x1, b2_x1)).clamp(0) * \
            (torch.min(b1_y2, b2_y2) - torch.max(b1_y1, b2_y1)).clamp(0)
    w1, h1 = b1_x2 - b1_x1, b1_y2 - b1_y1
    w2, h2 = b2_x2 - b2_x1, b2_y2 - b2_y1
    union = (w1 * h1 + 1e-16) + w2 * h2 - inter
    iou = inter / union
    cw = torch.max(b1_x2, b2_x2) - torch.min(b1_x1, b2_x1)
    ch = torch.max(b1_y2, b2_y2) - torch.min(b1_y1, b2_y1)
    c_area = cw * ch + 1e-16
    return iou - (c_area - union) / c_area


def build_targets(p, targets, anchor_vecs, iou_t):
    """utils.py:725-779 with use_all_anchors=True, reject=True -> (tcls, tbox, indices, av) per yolo layer."""
    nt = targets.shape[0]
    tcls, tbox, indices, av = [], [], [], []
    gain = torch.ones(6, device=targets.device)
    for i, anchors in enumerate(anchor_vecs):
        gain[2:] = torch.tensor(p[i].shape)[[3, 2, 3, 2]].float().to(targets.device)   # utils.py:742
        t, a = targets * gain, []
        gwh = t[:, 4:6]
        if nt:
            iou = wh_iou(anchors, gwh)
            na = anchors.shape[0]
            a = torch.arange(na, device=targets.device).view(-1, 1).repeat(1, nt).view(-1)   # utils.py:750 (anchor-major)
            t = t.repeat(na, 1)
            j = iou.view(-1) > iou_t                                               # utils.py:757
            t, a = t[j], a[j]
        b, c = t[:, :2].long().t()
        gxy = t[:, 2:4].clone()
        gwh = t[:, 4:6]
        gi, gj = gxy.long().t()                                                    # utils.py:764 (truncation)
        indices.append((b, a, gj, gi))
        gxy = gxy - gxy.floor()
        tbox.append(torch.cat((gxy, gwh), 1))
        av.append(anchors[a] if nt else anchors[:0])
        tcls.append(c)
    return tcls, tbox, indices, av


def compute_loss(p, targets, anchor_vecs, hyp, nc, gr=1.0):
    """utils.py:368-432 with red='mean', smooth_BCE(eps=0) -> (loss[1], items[4] = lbox, lobj, lcls, loss)."""
    dev = p[0].device
    lcls, lbox, lobj = torch.zeros(1, device=dev), torch.zeros(1, device=dev), torch.zeros(1, device=dev)
    tcls, tbox, indices, av = build_targets(p, targets, anchor_vecs, hyp['iou_t'])
    BCEcls = torch.nn.BCEWithLogitsLoss(pos_weight=torch.tensor([hyp['cls_pw']], device=dev), reduction='mean')
    BCEobj = torch.nn.BCEWithLogitsLoss(pos_weight=torch.tensor([hyp['obj_pw']], device=dev), reduction='mean')
    for i, pi in enumerate(p):
        b, a, gj, gi = indices[i]
        tobj = torch.zeros_like(pi[..., 0])
        nb = len(b)
        if nb:
            ps = pi[b, a, gj, gi]
            pxy = torch.sigmoid(ps[:, 0:2])
            pwh = torch.exp(ps[:, 2:4]).clamp(max=1E3) * av[i]
            pbox = torch.cat((pxy, pwh), 1)
            giou = giou_xywh(pbox.t(), tbox[i])
            lbox = lbox + (1.0 - giou).mean()
            tobj[b, a, gj, gi] = (1.0 - gr) + gr * giou.detach().clamp(0).type(tobj.dtype)   # utils.py:407
            if nc > 1:
                t = torch.full_like(ps[:, 5:], 0.0)
                t[range(nb), tcls[i]] = 1.0
                lcls = lcls + BCEcls(ps[:, 5:], t)
        lobj = lobj + BCEobj(pi[..., 4], tobj)
    lbox = lbox * hyp['giou']
    lobj = lobj * hyp['obj']
    lcls = lcls * hyp['cls']
    loss = lbox + lobj + lcls
    return loss, torch.cat((lbox, lobj, lcls, loss)).detach()


# ------------------------------------------------------------------------------------------------------------------
# quantisation -- utils/quantized/quantized_ptq_cos.py:14-113
# ------------------------------------------------------------------------------------------------------------------
def round_half_away(x):
    return torch.sign(x) * torch.floor(torch.abs(x) + 0.5)                          # ptq_cos.py:14-20


def pow2_scale(step, bits):
    return (2.0 ** step) / float(1 << (bits - 1))                                   # ptq_cos.py:32-41


def fake_quant(x, scale, bits):
    lo, hi = -(1 << (bits - 1)), (1 << (bits - 1)) - 1
    return torch.clamp(round_half_away(x / scale), lo, hi) * scale                  # ptq_cos.py:89-92


def cos_scale_search(x, bits):
    """ptq_cos.py:71-87: cosine similarity of x vs fake_quant(x) for steps i-5, i in range(bits+7); returns
    (argmax index i using the reference's strict '>' first-wins rule, list of similarities)."""
    sims = []
    best, best_i = -1.0, 0
    for i in range(bits + 7):
        q = fake_quant(x, pow2_scale(i - 5, bits), bits)
        cs = torch.cosine_similarity(x.view(-1), q.view(-1), dim=0)
        sims.append(float(cs))
        if cs > best:
            best, best_i = cs, i
    return best_i, sims
