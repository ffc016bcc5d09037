"""Distilled-data generation: drop-in for ``ZeroQ/distill_data.py`` (getDistilData), SURVEY.md section 8(f) rank 2.

The step immediately BEFORE the ``--distill_range`` path (main_cls.py:97-98, main_seg.py:119-120, main_ssd.py:193-194):
batches of synthetic images are optimised (Adam on the pixels, 1000 iterations, ReduceLROnPlateau, early break) until the
statistics of every BatchNorm INPUT match that layer's running mean / standard deviation (distill_data.py:75-227).

Same signature, same algorithm and same random-number consumption as the reference; what is GPU-native:

* the statistics-matching loss of every BatchNorm layer - per-(sample, channel) mean and unbiased std over H*W, two squared
  distances - is ONE fused forward kernel and ONE fused backward kernel (dfq_bnstat_loss_fwd / _bwd, csrc/distill.cu) instead
  of a dozen eager ops with full-size temporaries and their autograd replay;
* batches are independent optimisations: with torch.distributed initialised they are dealt round-robin to the ranks
  (one process per GPU) and all-gathered at the end - every rank draws the initial noise of ALL batches so the global RNG
  stream, and therefore batch i's starting point, is what a single process would have produced;
* the reference's per-iteration ``loss.item()`` (scheduler + early break need the value on the host) is kept: one sync per
  iteration is negligible next to the network's forward/backward.

The network's own forward/backward stays PyTorch (cuDNN); it is the model, not the path.
"""
import ctypes as C

import torch
import torch.nn as nn
import torch.optim as optim

from . import _lib


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _channel_stat(t, x, name):
    """A BatchNorm statistic as the kernels read it: [C] contiguous fp32 on x's device."""
    if t.device != x.device:
        raise _lib.DfqError("%s is on %s, the input on %s" % (name, t.device, x.device))
    if t.numel() != x.shape[1]:
        raise _lib.DfqError("%s has %d elements for %d channels" % (name, t.numel(), x.shape[1]))
    return t.detach().reshape(-1).to(torch.float32).contiguous()


class _BNStatLoss(torch.autograd.Function):
    """(x [N,C,H,W], bn_mean [C], bn_std [C]) -> tensor [2] = (own_loss(bn_mean, mean_hw x), own_loss(bn_std, std_hw(x+eps)))
    as distill_data.py:171-185 computes them; gradient w.r.t. x only."""

    @staticmethod
    def forward(ctx, x, bn_mean, bn_std, eps):
        lib = _lib.load()
        xc = x.detach().contiguous()
        n, c = xc.shape[0], xc.shape[1]
        bn_mean, bn_std = _channel_stat(bn_mean, xc, "bn_mean"), _channel_stat(bn_std, xc, "bn_std")
        hw = xc.numel() // (n * c)
        m = xc.new_empty((n * c,)); s = xc.new_empty((n * c,))
        loss = xc.new_empty((2,), dtype=torch.float64)
        with _lib.launch(xc) as st:
            _lib.check(lib.dfq_bnstat_loss_fwd(_ptr(xc), n, c, hw, _ptr(bn_mean), _ptr(bn_std), C.c_float(eps), _ptr(m), _ptr(s),
                                               _ptr(loss), st), "dfq_bnstat_loss_fwd")
        ctx.save_for_backward(xc, bn_mean, bn_std, m, s)
        ctx.eps = eps
        return loss.float()

    @staticmethod
    def backward(ctx, grad):
        lib = _lib.load()
        xc, bn_mean, bn_std, m, s = ctx.saved_tensors
        n, c = xc.shape[0], xc.shape[1]
        hw = xc.numel() // (n * c)
        gx = torch.empty_like(xc)
        g2 = grad.detach().float().contiguous()
        with _lib.launch(xc) as st:
            _lib.check(lib.dfq_bnstat_loss_bwd(_ptr(xc), _ptr(gx), n, c, hw, _ptr(bn_mean), _ptr(bn_std), C.c_float(ctx.eps), _ptr(m),
                                               _ptr(s), _ptr(g2), 0, st), "dfq_bnstat_loss_bwd")
        return gx, None, None, None


def bn_stat_loss(x, bn_mean, bn_std, eps=1e-6):
    """Fused (mean_loss, std_loss) of one BatchNorm input; falls back to the reference's formula where the kernel does not
    apply (1x1 spatial inputs use a different - memory-reinterpreting - view in the reference, distill_data.py:181-182)."""
    n, c = x.size(0), x.size(1)
    if x.is_cuda and x.dtype == torch.float32 and x.dim() >= 3 and x.numel() // (n * c) > 1:
        out = _BNStatLoss.apply(x, bn_mean, bn_std, eps)
        return out[0], out[1]
    flat = x.view(n, c, -1)
    tmp_mean = torch.mean(flat, dim=2)
    tmp_std = torch.std(flat + eps, dim=2) if flat.size(-1) != 1 else torch.std(x.view(c, -1) + eps, dim=1)
    own = lambda a, b: (a - b).norm() ** 2 / a.size(0)
    return own(bn_mean, tmp_mean), own(bn_std, tmp_std)


class _InputHook(object):
    """Forward hook keeping the input of a layer (distill_data.py:62-74)."""

    def __init__(self):
        self.inputs = None

    def hook(self, module, input, output):
        self.inputs = input

    def clear(self):
        self.inputs = None


def _initial_noise(batch_size, num_batch, max_value):
    """What iterating getRandomData's DataLoader yields for the first `num_batch` batches (ZeroQ/utils/data_utils.py:27-74):
    per sample ((randint(255) - 127) / 128) * max_value of shape [3, 224, 224] - the loader ignores `size` and
    `for_inception` - drawn sample by sample from the global RNG, after the one draw DataLoader.__iter__ takes for its
    base seed."""
    torch.empty((), dtype=torch.int64).random_()          # _BaseDataLoaderIter.__init__: base seed
    out = []
    for _ in range(num_batch):
        out.append(torch.stack([((torch.randint(high=255, size=(3, 224, 224)).float() - 127.) / 128.) * max_value
                                for _ in range(batch_size)]))
    return out


def getDistilData(teacher_model, dataset, batch_size, num_batch=1, bn_merged=False, for_inception=False, gpu=True,
                  value_range=[-10, 10], size=[224, 224], max_value=3., early_break_factor=1., group=None, iterations=1000):
    """
    Generate distilled data according to the BatchNorm statistics in the pretrained single-precision model.

    teacher_model: pretrained single-precision model
    dataset: the name of the dataset ('imagenet' or 'cifar10'; only selects the noise shape in the reference)
    batch_size: the batch size of generated distilled data
    num_batch: the number of batch of generated distilled data
    group / iterations: extensions (process group to spread the batches over; iteration cap, 1000 in the reference)
    """
    print("Start distilling data")
    if dataset not in ("imagenet", "cifar10"):
        raise NotImplementedError
    import torch.distributed as dist
    world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
    rank = dist.get_rank(group) if world > 1 else 0
    if dataset == "cifar10":
        torch.empty((), dtype=torch.int64).random_()
        noise = [torch.stack([((torch.randint(high=255, size=(3, 32, 32)).float() - 127.) / 128.) * max_value
                              for _ in range(batch_size)]) for _ in range(num_batch)]
    else:
        noise = _initial_noise(batch_size, num_batch, max_value)
    eps = 1e-6
    if gpu:
        _lib.require_cuda()
        teacher_model = teacher_model.cuda()
    teacher_model = teacher_model.eval()
    dev = next(teacher_model.parameters()).device
    hooks, handles, bn_stats = [], [], []
    layers = sum(1 for m in teacher_model.modules() if isinstance(m, nn.BatchNorm2d))
    for m in teacher_model.modules():
        if isinstance(m, nn.BatchNorm2d):
            hook = _InputHook()
            hooks.append(hook)
            handles.append(m.register_forward_hook(hook.hook))
            if not bn_merged:
                bn_stats.append((m.running_mean.detach().clone().flatten().to(dev).contiguous(),
                                 torch.sqrt(m.running_var + eps).detach().clone().flatten().to(dev).contiguous()))
            else:
                bn_stats.append((m.fake_bias.detach().clone().flatten().to(dev).contiguous(),
                                 m.fake_weight.detach().clone().flatten().to(dev).contiguous()))
    assert len(hooks) == len(bn_stats)
    input_mean = torch.zeros(3, device=dev)
    input_std = torch.ones(3, device=dev)
    refined = [None] * num_batch
    try:
        for i in range(num_batch):
            if i % world != rank:
                continue
            data = noise[i].to(dev)
            data.requires_grad = True
            optimizer = optim.Adam([data], lr=0.1)
            scheduler = optim.lr_scheduler.ReduceLROnPlateau(optimizer, min_lr=1e-7, patience=100)
            for it in range(iterations):
                teacher_model.zero_grad()
                optimizer.zero_grad()
                for hook in hooks:
                    hook.clear()
                teacher_model(data.clamp(value_range[0], value_range[1]))
                mean_loss = 0
                std_loss = 0
                for (bn_mean, bn_std), hook in zip(bn_stats, hooks):
                    lm, ls = bn_stat_loss(hook.inputs[0], bn_mean, bn_std, eps)
                    mean_loss = mean_loss + lm
                    std_loss = std_loss + ls
                # the statistics of the images themselves against N(0, 1) (distill_data.py:186-192): no eps here
                flat = data.view(data.size(0), 3, -1)
                own = lambda a, b: (a - b).norm() ** 2 / a.size(0)
                mean_loss = mean_loss + own(torch.mean(flat, dim=2), input_mean.view(1, 3))
                std_loss = std_loss + own(torch.std(flat, dim=2), input_std.view(1, 3))
                total_loss = mean_loss + std_loss
                total_loss.backward()
                optimizer.step()
                value = total_loss.item()
                scheduler.step(value)
                if value <= (layers + 1) * early_break_factor:      # early stop to prevent overfitting
                    break
            print("{} out of {} distilled.".format(i + 1, num_batch))
            refined[i] = data.detach().clone().clamp(value_range[0], value_range[1])
    finally:
        for h in handles:
            h.remove()
    if world > 1:
        for i in range(num_batch):
            buf = refined[i] if refined[i] is not None else torch.empty_like(noise[i], device=dev)
            dist.broadcast(buf, src=i % world, group=group)
            refined[i] = buf
    return refined
