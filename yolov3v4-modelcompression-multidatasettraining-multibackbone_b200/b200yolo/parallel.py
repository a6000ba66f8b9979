"""Data parallelism for the Darknet hot path: one process per GPU, ONE gradient all-reduce per step.

Reference: train.py:93-107 (NCCL process group), :219-221 (DistributedDataParallel, find_unused_parameters=True),
DDP's bucketed all-reduce (SUM, then / world) overlapped with backward, rank-0 buffer broadcast every forward
(broadcast_buffers=True), optimiser groups train.py:125-144 (weight decay on 'Conv2d.weight' only).

Here all parameters live in one flat fp32 buffer and all gradients in another (the training plan writes weight
gradients straight into their slice), so the exchange step is exactly one `all_reduce(flat_grad, SUM)` over
NCCL/NVLink and the 1/world factor is folded into the fused optimiser kernel.  Semantics kept from DDP:
  * reduced gradient = mean over ranks of the per-rank gradients (each rank's loss uses its own shard),
  * BatchNorm statistics are per replica; running buffers follow rank 0 (broadcast before each forward),
  * parameters are broadcast from rank 0 at construction.
`torch.distributed` provides the communicator (backend "nccl" on GPUs, "gloo" in the CPU tests).
"""
import torch
import torch.distributed as dist


def _is_decay_param(name):
    """train.py:126-133: pg1 (weight decay) = names containing 'Conv2d.weight'; '.bias' -> pg2; rest -> pg0."""
    return ('.bias' not in name) and ('Conv2d.weight' in name)


class FlatDataParallel:
    def __init__(self, model, process_group=None, broadcast_buffers=True):
        self.module = model
        self.pg = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(process_group) if dist.is_initialized() else 0
        self.broadcast_buffers = broadcast_buffers
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        decay = [(n, p) for n, p in named if _is_decay_param(n)]
        other = [(n, p) for n, p in named if not _is_decay_param(n)]
        self.names = [n for n, _ in decay + other]
        self.params = [p for _, p in decay + other]
        self.n_decay = sum(p.numel() for _, p in decay)
        total = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat_param = torch.empty(total, dtype=torch.float32, device=dev)
        self.flat_grad = torch.zeros(total, dtype=torch.float32, device=dev)
        self.flat_mom = torch.zeros(total, dtype=torch.float32, device=dev)
        self.grad_views = {}
        off = 0
        with torch.no_grad():
            for p in self.params:
                n = p.numel()
                self.flat_param[off:off + n].copy_(p.detach().reshape(-1))
                p.data = self.flat_param[off:off + n].view_as(p)          # parameters become views of the flat buffer
                gv = self.flat_grad[off:off + n].view_as(p)
                p.grad = gv
                self.grad_views[id(p)] = gv
                off += n
        # BatchNorm running statistics become views of ONE flat buffer as well, so that "rank 0's buffers win" (DDP
        # broadcast_buffers, N3) is a single broadcast per forward instead of a cat + 2 copies per BatchNorm layer
        self.buffers = [b for b in model.buffers() if b.dtype.is_floating_point]
        nb = sum(b.numel() for b in self.buffers)
        self.flat_buf = torch.empty(nb, dtype=torch.float32, device=dev) if nb else None
        off = 0
        with torch.no_grad():
            for b in self.buffers:
                n = b.numel()
                self.flat_buf[off:off + n].copy_(b.detach().reshape(-1).float())
                b.data = self.flat_buf[off:off + n].view_as(b)
                off += n
        self.has_momentum = False        # flat_mom holds a momentum buffer: set by the SGD step or a loaded state
        self._l1 = None
        self._sgd = None
        if self.world > 1:
            dist.broadcast(self.flat_param, src=0, group=self.pg)           # N2: parameters from rank 0
            self._broadcast_buffers()
        eng = getattr(model, 'engine', None)
        if callable(eng):
            model.engine().invalidate()
        model._b2y_grad_sink = self.grad_views     # the training plan writes gradients straight into flat_grad

    # DDP-like attribute forwarding so that utils.utils.compute_loss(model=wrapper) keeps working
    def __getattr__(self, name):
        return getattr(self.__dict__['module'], name)

    def _broadcast_buffers(self):
        if self.flat_buf is None:
            return
        dist.broadcast(self.flat_buf, src=0, group=self.pg)

    def __call__(self, x, *a, **k):
        if self.world > 1 and self.broadcast_buffers and self.module.training:
            self._broadcast_buffers()                                       # N3: rank-0 running stats win
        return self.module(x, *a, **k)

    def zero_grad(self):
        self.flat_grad.zero_()

    def accumulate(self):
        """Gradient accumulation over micro-batches (train.py:437-447, `accumulate = 64 / batch_size`): the training plan
        OVERWRITES the flat gradient buffer on every backward (its kernels write, they do not add), so call this after
        each micro-batch's backward; reduce_gradients() / step() then use the sum.  Without it, two backward calls
        before a step keep only the last one."""
        if getattr(self, '_acc', None) is None:
            self._acc = self.flat_grad.clone()
        else:
            self._acc.add_(self.flat_grad)

    def reduce_gradients(self, async_op=False):
        """The single exchange step of the data-parallel path (N4): SUM over ranks; the mean is taken in step()."""
        if getattr(self, '_acc', None) is not None:
            self.flat_grad.copy_(self._acc)
            self._acc = None
        if self.world > 1:
            return dist.all_reduce(self.flat_grad, op=dist.ReduceOp.SUM, group=self.pg, async_op=async_op)
        return None

    def averaged_gradients(self):
        """flat gradient divided by world (what DDP leaves in .grad) -- used by the tests."""
        return self.flat_grad / float(self.world)

    def enable_ema(self, decay=0.9999):
        """Model EMA (utils/torch_utils.py:141-183, train.py --ema) fused into the optimiser pass: flat copies of the
        parameters and of the BatchNorm running buffers, decay ramp d(t) = decay * (1 - exp(-t / 2000))."""
        import math
        self.ema_param = self.flat_param.clone()
        self.ema_buf = self.flat_buf.clone() if self.flat_buf is not None else None
        self.ema_updates = 0
        self._ema_decay = lambda t: decay * (1 - math.exp(-t / 2000))

    def ema_state_dict(self):
        """name -> EMA tensor for every parameter and floating-point buffer (views of the flat EMA buffers)."""
        out, off = {}, 0
        for n, p in zip(self.names, self.params):
            out[n] = self.ema_param[off:off + p.numel()].view_as(p)
            off += p.numel()
        off = 0
        names = [n for n, b in self.module.named_buffers() if b.dtype.is_floating_point]
        for n, b in zip(names, self.buffers):
            out[n] = self.ema_buf[off:off + b.numel()].view_as(b)
            off += b.numel()
        return out

    def set_bn_sparsity(self, prune_idx, s):
        """Network-slimming sparsity training (train.py -sr --s, :444-445; prune_utils.py:133-138 BNOptimizer.updateBN):
        from now on the optimiser step adds s * sign(gamma) to the (averaged) gradient of the BatchNorm scale of every
        module_list[idx] in prune_idx, in the same launch as the update.  Kept on the host: an int64 CPU table of the
        (offset, length) rows of those scales in the flat buffers, and s.  s = 0 or an empty list switches it off."""
        offsets, off = {}, 0
        for p in self.params:
            offsets[id(p)] = off
            off += p.numel()
        rows = []
        for idx in (prune_idx if s else []):
            bn = self.module.module_list[idx][1]
            rows.append((offsets[id(bn.weight)], bn.weight.numel()))
        self._l1 = (torch.tensor(rows, dtype=torch.int64).reshape(-1, 2), float(s)) if rows else None

    def step(self, lr, momentum=0.937, weight_decay=0.000484, nesterov=True):
        """Nesterov SGD with one lr and momentum, weight decay on the 'Conv2d.weight' parameters only: a
        b200yolo.optim.FlatSGD step over two groups, those parameters and the rest (+ BatchNorm-L1 and EMA when enabled),
        in one launch."""
        assert nesterov, "the fused kernel implements the reference's nesterov=True configuration"
        if self._sgd is None:
            from .optim import FlatSGD
            nd = sum(map(_is_decay_param, self.names))        # the decayed parameters come first in the flat layout
            self._sgd = FlatSGD(self, [{'params': self.params[:nd]}, {'params': self.params[nd:]}], lr, momentum)
        for group, wd in zip(self._sgd.param_groups, (weight_decay, 0.0)):
            group.update(lr=lr, momentum=momentum, weight_decay=wd)
        self._sgd.step()
