"""Darknet(cfg) model API of the reference (models.py) on top of the H100-native engine.

Public surface kept from the reference (file:line are the reference's models.py):
    create_modules :11-347      YOLOLayer :350-437      Darknet :440-580      get_yolo_layers :583
    load_darknet_weights :587-735      save_weights :738-782      convert :785-813      attempt_download :816-843

The module tree (nn.ModuleList of nn.Sequential{Conv2d, BatchNorm2d, activation} / Shortcut / FeatureConcat /
Upsample / MaxPool2d / YOLOLayer), parameter names, state_dict keys and the Darknet .weights layout are exactly
the reference's, so checkpoints, optimiser grouping (train.py:125-133) and the pruning scripts' indexing
(module_list[i][0] / [1]) keep working.  What changes is *execution*: Darknet.forward does not walk the modules
with ATen/cuDNN calls; it hands the graph to b200yolo.engine, which runs fused conv+BN+activation(+shortcut)
wgmma kernels on NHWC fp16 activations and the fp32 YOLO decode kernel.
"""
from utils.google_utils import *  # noqa: F401,F403
from utils.parse_config import *  # noqa: F401,F403
from utils.layers import *  # noqa: F401,F403
from utils import torch_utils
import copy

ONNX_EXPORT = False

_ACTIVATIONS = {
    'leaky': lambda slope: nn.LeakyReLU(slope, inplace=True),
    'relu6': lambda slope: ReLU6(),
    'h_swish': lambda slope: HardSwish(),
    'relu': lambda slope: nn.ReLU(),
    'mish': lambda slope: Mish(),
}


def _quantized_layers():
    """Lazy import of the quantised layer zoo (utils/quantized/*), only needed for quantized != -1."""
    from utils.quantized import quantized_google, quantized_ptq_cos, quantized_TPSQ
    return quantized_google, quantized_ptq_cos, quantized_TPSQ


def _conv_block(mdef, in_ch, depthwise, quantized, qkw, maxabsscaler, index):
    """[convolutional] / [depthwise] -> nn.Sequential with children named Conv2d|DepthWise2d, BatchNorm2d, activation."""
    bn = int(mdef['batch_normalize'])
    filters = int(mdef['filters'])
    k = int(mdef['size'])
    pad = (k - 1) // 2 if int(mdef['pad']) else 0
    stride = int(mdef['stride'])
    groups = in_ch if depthwise else (mdef['groups'] if 'groups' in mdef else 1)
    child = 'DepthWise2d' if depthwise else 'Conv2d'
    seq = nn.Sequential()
    # google QAT keeps [depthwise] blocks in float: the reference's quantized == 1 branch is overwritten by its float
    # `else` (reference models.py:120-184), so the block is Conv2d(groups=C) + BatchNorm2d + activation
    if quantized in (1, 2, 3) and not (depthwise and quantized == 1):
        g, c, t = _quantized_layers()
        name = "{:04d}".format(index) + "_" + mdef['type'][:4]
        common = dict(in_channels=in_ch, out_channels=filters, kernel_size=k, stride=stride, padding=pad, groups=groups,
                      bias=not bn, a_bits=qkw['a_bit'], w_bits=qkw['w_bit'], bn=bn, activate=mdef['activation'],
                      quantizer_output=qkw['quantizer_output'], maxabsscaler=maxabsscaler)
        if quantized == 1:
            layer = g.BNFold_QuantizedConv2d_For_FPGA(steps=qkw['steps'], reorder=qkw['reorder'], TM=qkw['TM'],
                                                      TN=qkw['TN'], name=name, layer_idx=qkw['layer_idx'], **common)
        elif quantized == 2:
            layer = t.TPSQ_BNFold_QuantizedConv2d_For_FPGA(steps=qkw['steps'], **common)
        else:
            layer = c.BNFold_COSPTQuantizedConv2d_For_FPGA(reorder=qkw['reorder'], TM=qkw['TM'], TN=qkw['TN'],
                                                           name=name, layer_idx=qkw['layer_idx'], **common)
        seq.add_module(child, layer)
        return seq, filters
    seq.add_module(child, nn.Conv2d(in_channels=in_ch, out_channels=filters, kernel_size=k, stride=stride, padding=pad,
                                    groups=groups, bias=not bn))
    if bn:
        seq.add_module('BatchNorm2d', nn.BatchNorm2d(filters, momentum=0.1))
    make_act = _ACTIVATIONS.get(mdef['activation'])
    if make_act is not None:
        seq.add_module('activation', make_act(0.25 if maxabsscaler else 0.1))
    return seq, filters


def create_modules(module_defs, img_size, cfg, quantized, quantizer_output, layer_idx, reorder, TM, TN, a_bit=8,
                   w_bit=8, steps=0, is_gray_scale=False, maxabsscaler=False, shortcut_way=-1):
    """module_defs (with [net] first; it is popped, like the reference does) -> (nn.ModuleList, routs bool list)."""
    img_size = [img_size] * 2 if isinstance(img_size, int) else img_size
    module_defs.pop(0)
    output_filters = [1 if is_gray_scale else 3]
    module_list = nn.ModuleList()
    routs = []
    yolo_index = -1
    qkw = dict(a_bit=a_bit, w_bit=w_bit, steps=steps, quantizer_output=quantizer_output, reorder=reorder, TM=TM, TN=TN,
               layer_idx=layer_idx)
    filters = output_filters[-1]
    i = -1
    for i, mdef in enumerate(module_defs):
        kind = mdef['type']
        modules = nn.Sequential()
        if kind in ('convolutional', 'depthwise'):
            modules, filters = _conv_block(mdef, output_filters[-1], kind == 'depthwise', quantized, qkw, maxabsscaler,
                                           i)
        elif kind == 'BatchNorm2d':
            filters = output_filters[-1]
            modules = nn.BatchNorm2d(filters, momentum=0.03, eps=1E-4)
            if i == 0 and filters == 3:  # ImageNet statistics for an RGB input-normalisation layer
                modules.running_mean = torch.tensor([0.485, 0.456, 0.406])
                modules.running_var = torch.tensor([0.0524, 0.0502, 0.0506])
        elif kind == 'maxpool':
            k, stride = mdef['size'], mdef['stride']
            pool = nn.MaxPool2d(kernel_size=k, stride=stride, padding=(k - 1) // 2)
            if k == 2 and stride == 1:  # yolov3-tiny
                modules.add_module('ZeroPad2d', nn.ZeroPad2d((0, 1, 0, 1)))
                modules.add_module('MaxPool2d', pool)
            else:
                modules = pool
        elif kind == 'se':
            if 'filters' in mdef:
                filters = int(mdef['filters'])
            modules.add_module('se', SE(channel=filters))
            if 'reduction' in mdef:
                modules.add_module('se', SE(output_filters[-1], reduction=int(mdef['reduction'])))
        elif kind == 'upsample':
            modules = nn.Upsample(scale_factor=mdef['stride'])
        elif kind == 'route':
            layers = mdef['layers']
            filters = sum(output_filters[l + 1 if l > 0 else l] for l in layers)
            grouped = 'groups' in mdef
            if grouped:
                filters = filters // 2
            routs.extend([i + l if l < 0 else l for l in layers])
            if quantized == -1:
                modules = FeatureConcat(layers=layers, groups=grouped)
            else:
                g, c, _ = _quantized_layers()
                cls = c.COSPTQuantizedFeatureConcat if quantized == 3 else g.QuantizedFeatureConcat
                modules = cls(layers=layers, groups=grouped, bits=a_bit, quantizer_output=quantizer_output,
                              reorder=reorder, TM=TM, TN=TN, name="{:04d}".format(i) + "_" + kind[:4],
                              layer_idx=layer_idx)
        elif kind == 'shortcut':
            layers = mdef['from']
            filters = output_filters[-1]
            routs.extend([i + l if l < 0 else l for l in layers])
            weighted = 'weights_type' in mdef
            if quantized in (-1, 2):
                modules = Shortcut(layers=layers, weight=weighted)
            else:
                g, c, _ = _quantized_layers()
                table = {(3, 1): c.COSPTQuantizedShortcut_min, (3, 2): c.COSPTQuantizedShortcut_max,
                         (1, 1): g.QuantizedShortcut_min, (1, 2): g.QuantizedShortcut_max}
                cls = table.get((quantized, shortcut_way))
                if cls is not None:  # (shortcut_way not in {1,2} leaves an empty Sequential, like the reference)
                    modules = cls(layers=layers, weight=weighted, bits=a_bit, quantizer_output=quantizer_output,
                                  reorder=reorder, TM=TM, TN=TN, name="{:04d}".format(i) + "_" + kind[:4],
                                  layer_idx=layer_idx)
        elif kind == 'reorg3d':
            pass
        elif kind == 'yolo':
            yolo_index += 1
            stride = [32, 16, 8]
            if any(tag in cfg for tag in ('panet', 'yolov4', 'cd53')) and 'yolov4-tiny' not in cfg:
                stride = stride[::-1]
            layers = mdef['from'] if 'from' in mdef else []
            modules = YOLOLayer(anchors=mdef['anchors'][mdef['mask']], nc=mdef['classes'], img_size=img_size,
                                yolo_index=yolo_index, layers=layers, stride=stride[yolo_index],
                                quantizer_output=quantizer_output)
            # prior-probability bias init of the preceding head conv (obj ~ 0.01, cls ~ 0.6/nc)
            try:
                with torch.no_grad():
                    j = layers[yolo_index] if 'from' in mdef else -1
                    head = module_list[j][0]
                    b = head.bias[:modules.no * modules.na].view(modules.na, -1)
                    b[:, 4] = b[:, 4] - 4.5
                    b[:, 5:] = b[:, 5:] + math.log(0.6 / (modules.nc - 0.99))
                    head.bias = torch.nn.Parameter(head.bias.detach(), requires_grad=head.bias.requires_grad)
            except Exception:
                print('WARNING: smart bias initialization failure.')
        else:
            print('Warning: Unrecognized Layer Type: ' + kind)
        module_list.append(modules)
        output_filters.append(filters)

    routs_binary = [False] * (i + 1)
    for r in routs:
        routs_binary[r] = True
    return module_list, routs_binary


class YOLOLayer(nn.Module):
    """Detection head bookkeeping: anchors / stride / grid sizes.  The tensor math of the reference's forward
    (view+permute, sigmoid/exp decode) is the b2y_yolo_decode kernel; `forward` here serves module-level calls on
    an NCHW fp32 head output and uses the same kernel."""

    def __init__(self, anchors, nc, img_size, yolo_index, layers, stride, quantizer_output=False):
        super().__init__()
        self.anchors = torch.Tensor(anchors)
        self.index = yolo_index
        self.layers = layers
        self.stride = stride
        self.nl = len(layers)
        self.na = len(anchors)
        self.nc = nc
        self.no = nc + 5
        self.nx, self.ny, self.ng = 0, 0, 0
        self.anchor_vec = self.anchors / self.stride
        self.anchor_wh = self.anchor_vec.view(1, self.na, 1, 1, 2)
        self.quantizer_output = quantizer_output

    def create_grids(self, ng=(13, 13), device='cpu'):
        self.nx, self.ny = ng
        self.ng = torch.tensor(ng, dtype=torch.float)
        if not self.training:
            yv, xv = torch.meshgrid([torch.arange(self.ny, device=device), torch.arange(self.nx, device=device)],
                                    indexing='ij')
            self.grid = torch.stack((xv, yv), 2).view((1, 1, self.ny, self.nx, 2)).float()
        if self.anchor_vec.device != device:
            self.anchor_vec = self.anchor_vec.to(device)
            self.anchor_wh = self.anchor_wh.to(device)

    def forward(self, p, out=None):
        from b200yolo import ops
        if not p.is_cuda:
            raise RuntimeError("YOLOLayer.forward runs on the CUDA device only (no CPU fallback)")
        bs, _, ny, nx = p.shape
        self.create_grids((nx, ny), p.device)
        raw = p.float().permute(0, 2, 3, 1).contiguous()
        io = None if self.training else torch.empty((bs, self.na * ny * nx, self.no), device=p.device)
        io, pp = ops.yolo_decode(raw, self.na, self.no, self.anchors.to(p.device), self.stride, io=io)
        return pp if self.training else (io, pp)


class Darknet(nn.Module):
    """YOLOv3/v4 detector built from a Darknet cfg (path or list of block dicts)."""

    def __init__(self, cfg, img_size=(416, 416), verbose=False, quantized=-1, a_bit=8, w_bit=8,
                 quantizer_output=False, layer_idx=-1, reorder=False, TM=32, TN=32, steps=0, is_gray_scale=False,
                 maxabsscaler=False, shortcut_way=-1, FPGA=False):
        super().__init__()
        if isinstance(cfg, str):
            self.module_defs = parse_model_cfg(cfg)
        elif isinstance(cfg, list):
            self.module_defs = cfg
        self.quantized = quantized
        self.a_bit = a_bit
        self.w_bit = w_bit
        self.quantizer_output = quantizer_output
        self.layer_idx = layer_idx
        self.reorder = reorder
        self.TM = TM
        self.TN = TN
        self.is_gray_scale = is_gray_scale
        self.maxabsscaler = maxabsscaler
        self.FPGA = FPGA  # accepted and ignored: detect.py:26 / convert_FPGA.py:18 pass it
        self.hyperparams = copy.deepcopy(self.module_defs[0])
        self.module_list, self.routs = create_modules(
            self.module_defs, img_size, cfg, quantized=quantized, quantizer_output=quantizer_output, reorder=reorder,
            TM=TM, TN=TN, layer_idx=layer_idx, a_bit=a_bit, w_bit=w_bit, steps=steps, is_gray_scale=is_gray_scale,
            maxabsscaler=maxabsscaler, shortcut_way=shortcut_way)
        self.yolo_layers = get_yolo_layers(self)
        self.version = np.array([0, 2, 5], dtype=np.int32)
        self.seen = np.array([0], dtype=np.int64)
        self.keep_features = None  # None: keep in training, drop in eval (see b200yolo/engine.py)
        self._engine = None
        if self.quantized == -1:
            self.info(verbose)

    # ---- execution -------------------------------------------------------------------------------------------
    def engine(self):
        if self._engine is None:
            from b200yolo.engine import Engine
            object.__setattr__(self, '_engine', Engine(self))
        return self._engine

    def __deepcopy__(self, memo):
        eng = self.__dict__.get('_engine')
        object.__setattr__(self, '_engine', None)
        try:
            cls = self.__class__
            new = cls.__new__(cls)
            memo[id(self)] = new
            for k, v in self.__dict__.items():
                object.__setattr__(new, k, copy.deepcopy(v, memo))
        finally:
            object.__setattr__(self, '_engine', eng)
        return new

    def __getstate__(self):
        state = dict(self.__dict__)
        state['_engine'] = None  # device buffers / CUDA graphs are rebuilt lazily
        return state

    def forward(self, x, augment=False):
        if not augment:
            return self.forward_once(x)
        img_size = x.shape[-2:]
        s = [0.83, 0.67]
        y = []
        for xi in (x, torch_utils.scale_img(x.flip(3), s[0], same_shape=False),
                   torch_utils.scale_img(x, s[1], same_shape=False)):
            y.append(self.forward_once(xi)[0])
        y[1][..., :4] /= s[0]
        y[1][..., 0] = img_size[1] - y[1][..., 0]
        y[2][..., :4] /= s[1]
        return torch.cat(y, 1), None

    def forward_once(self, x, augment=False, verbose=False):
        if not x.is_cuda:
            raise RuntimeError("Darknet.forward runs on a CUDA (sm_90a) device only: the H100 engine has no CPU "
                               "fallback. Move the model and the input to the GPU.")
        return self.engine().forward(x)

    def fuse(self):
        """Fold every BatchNorm2d into its Conv2d at module level (children become '0','1' like the reference)."""
        print('Fusing layers...')
        fused_list = nn.ModuleList()
        for a in list(self.children())[0]:
            if isinstance(a, nn.Sequential):
                for i, b in enumerate(a):
                    if isinstance(b, nn.modules.batchnorm.BatchNorm2d):
                        conv = a[i - 1]
                        a = nn.Sequential(torch_utils.fuse_conv_and_bn(conv, b), *list(a.children())[i + 1:])
                        break
            fused_list.append(a)
        self.module_list = fused_list
        object.__setattr__(self, '_engine', None)

    def info(self, verbose=False):
        torch_utils.model_info(self, verbose)


def _invalidate_engine(model):
    eng = model.__dict__.get('_engine')
    if eng is not None:
        eng.invalidate()


def get_yolo_layers(model):
    return [i for i, m in enumerate(model.module_list) if m.__class__.__name__ == 'YOLOLayer']


# ---- Darknet binary weights ------------------------------------------------------------------------------------
# header: int32[3] version, int64 seen; then per block (little-endian fp32):
#   conv+bn : bn.bias, bn.weight, bn.running_mean, bn.running_var, conv.weight
#   conv    : conv.bias, conv.weight
#   se      : fc1.weight, fc2.weight
def _bn_slots(block, quant):
    head = block[0]
    if quant and hasattr(head, 'gamma'):  # quantised convs keep the BN parameters on the conv module itself
        return [head.beta, head.gamma, head.running_mean, head.running_var]
    bn = block[1]
    return [bn.bias, bn.weight, bn.running_mean, bn.running_var]


def _weight_slots(mdef, block, quant=False):
    kind = mdef['type']
    if kind in ('convolutional', 'depthwise'):
        head = block[0]
        if mdef['batch_normalize']:
            return _bn_slots(block, quant) + [head.weight]
        return [head.bias, head.weight]
    if kind == 'se':
        fc = block[0].fc
        return [fc[0].weight, fc[2].weight]
    return []


def load_darknet_weights(self, weights, cutoff=-1, pt=False, quant=False):
    file = Path(weights).name
    if file == 'darknet53.conv.74':
        cutoff = 75
    elif file == 'yolov3-tiny.conv.15':
        cutoff = 15
    with open(weights, 'rb') as f:
        self.version = np.fromfile(f, dtype=np.int32, count=3)
        self.seen = np.fromfile(f, dtype=np.int64, count=1)
        blob = np.fromfile(f, dtype=np.float32)
    skip_coco_head = pt and os.path.basename(file).split('.')[-1] == 'weights'
    ptr = 0
    for i, (mdef, block) in enumerate(zip(self.module_defs[:cutoff], self.module_list[:cutoff])):
        if mdef['type'] == 'convolutional' and not mdef['batch_normalize'] and skip_coco_head:
            # COCO-pretrained file, custom class count: step over the 255-filter head
            ptr += 255 + int(self.module_defs[i - 1]["filters"]) * 255
            continue
        for slot in _weight_slots(mdef, block, quant):
            n = slot.numel()
            slot.data.copy_(torch.from_numpy(blob[ptr:ptr + n]).view_as(slot))
            ptr += n
    assert ptr == len(blob)
    _invalidate_engine(self)


def save_weights(self, path='model.weights', cutoff=-1):
    with open(path, 'wb') as f:
        self.version.tofile(f)
        self.seen.tofile(f)
        for mdef, block in zip(self.module_defs[:cutoff], self.module_list[:cutoff]):
            for slot in _weight_slots(mdef, block, quant=True):
                slot.data.cpu().numpy().tofile(f)


def convert(cfg='cfg/yolov3-spp.cfg', weights='weights/yolov3-spp.weights'):
    """.pt <-> .weights by file extension."""
    model = Darknet(cfg)
    if weights.endswith('.pt'):
        model.load_state_dict(torch.load(weights, map_location='cpu')['model'])
        target = weights.rsplit('.', 1)[0] + '.weights'
        save_weights(model, path=target, cutoff=-1)
        print("Success: converted '%s' to '%s'" % (weights, target))
    elif weights.endswith('.weights'):
        load_darknet_weights(model, weights)
        chkpt = {'epoch': -1, 'best_fitness': None, 'training_results': None, 'model': model.state_dict(),
                 'optimizer': None}
        target = weights.rsplit('.', 1)[0] + '.pt'
        torch.save(chkpt, target)
        print("Success: converted '%s' to '%s'" % (weights, target))
    else:
        print('Error: extension not supported.')


def attempt_download(weights):
    """The reference fetches missing weight files from Google Drive / pjreddie.com; this box has no network, so a
    missing file is reported instead (same exception type and message head as the reference)."""
    weights = weights.strip().replace("'", '')
    if len(weights) > 0 and not os.path.isfile(weights):
        raise Exception(weights + ' missing, try downloading from '
                        'https://drive.google.com/open?id=1LezFG5g3BCW6iYaV89B2i64cqEUZD7e0')
