"""Autograd glue of the training path (ctn_convtasnet_fwd_train / ctn_convtasnet_bwd, ctn_causal_fwd_train / ctn_causal_bwd
for causal models, ctn_multichannel_fwd_train / ctn_multichannel_bwd for in_channels > 1 and ctn_softmax_fwd_train /
ctn_softmax_bwd for softmax masks; include/ctn_b200.h).

The reference trains with plain autograd over its nn.Module graph (egs/wsj0-mix/common/src/driver.py:146-150:
``estimated = model(mixture); loss, _ = pit_criterion(estimated, sources); loss.backward()``).  Here the whole
model is ONE autograd node: the forward keeps the per-block activations in a device buffer owned by the node, the
backward is one C call that fills the gradients of all parameter tensors.  Gradients come back as views of one flat
zero-initialised buffer (the natural bucket for the data-parallel all-reduce, see ctn_b200/dist.py).

Only the softmax step takes a mixture that requires grad, and returns its gradient: the ORPIT fine-tune step feeds an estimate
back in as the next stage's mixture (egs/wsj0-mix/orpit_conv-tasnet/src/adhoc_driver.py, FinetuneTrainer.run_one_epoch_train)
and calls backward once over all stages.  So that clip + Adam still see one flat bucket, the softmax nodes of one backward pass
share it: the first to run owns the bucket, each later one adds its gradients into it in place."""
import ctypes as C

import torch

from .. import _native as N

TOP_FIELDS = N.TOP_FIELDS


def param_list(model):
    """[(slot, tensor-or-None)] in a fixed order; slot = top-level field name or (block index, block field name)."""
    return model.separator.param_slots(enc_w=model.encoder.conv1d.weight, dec_w=model.decoder.conv_transpose1d.weight)


class _Entry:
    """the three C entry points of a training step, by name in _native"""

    def __init__(self, workspace_bytes, fwd, bwd, multichannel=False, mixture_grad=False):
        self.WORKSPACE_BYTES, self.FWD, self.BWD = workspace_bytes, fwd, bwd
        self.multichannel = multichannel  # x (B, C, T) -> out (B, S, C, T); otherwise x (B, 1, T) -> out (B, S, T)
        self.mixture_grad = mixture_grad  # BWD takes a nullable d_x after d_out, and the nodes of one backward pass share a bucket


GLN = _Entry("ctn_train_workspace_bytes", "ctn_convtasnet_fwd_train", "ctn_convtasnet_bwd")
CAUSAL = _Entry("ctn_causal_train_workspace_bytes", "ctn_causal_fwd_train", "ctn_causal_bwd")
MULTICHANNEL = _Entry("ctn_multichannel_train_workspace_bytes", "ctn_multichannel_fwd_train", "ctn_multichannel_bwd", multichannel=True)
SOFTMAX = _Entry("ctn_softmax_train_workspace_bytes", "ctn_softmax_fwd_train", "ctn_softmax_bwd", mixture_grad=True)


def train_entry(model):
    """The training step a ConvTasNet runs under autograd, or NotImplementedError for a model that trains nowhere.  A softmax model
    without softmax_training takes the sigmoid step, and a causal softmax model with causal_training the causal step: their C
    entries refuse the mask."""
    if model.in_channels > 1:
        if not model.multichannel_training:
            raise NotImplementedError("multichannel models (in_channels > 1) train natively only with model.multichannel_training = True "
                                      "(ctn_multichannel_fwd_train / ctn_multichannel_bwd); without it they are forward only: call "
                                      "under torch.no_grad()")
        if model.causal or model.separator.mask_softmax:
            raise NotImplementedError("multichannel training is built for non-causal models with a sigmoid mask; causal or softmax "
                                      "multichannel models are forward only: call under torch.no_grad()")
        return MULTICHANNEL
    if model.separator.mask_softmax and model.softmax_training:
        if model.causal:
            raise NotImplementedError("softmax-mask training is built for non-causal monaural models (ctn_softmax_fwd_train / "
                                      "ctn_softmax_bwd); causal or multichannel softmax models are forward only: call under "
                                      "torch.no_grad()")
        return SOFTMAX
    if model.causal:
        if not model.causal_training:
            raise NotImplementedError("causal (cLN) models train natively only with model.causal_training = True (ctn_causal_fwd_train / "
                                      "ctn_causal_bwd); without it they are forward only: call under torch.no_grad()")
        return CAUSAL
    return GLN


class TrainFn(torch.autograd.Function):
    """The whole model as one autograd node over the training step `entry` (an _Entry)."""

    @staticmethod
    def forward(ctx, entry, model, x, *tensors):
        dev = N.require_cuda(x)
        B, Cin, T = x.shape
        slots = [s for s, _ in param_list(model)]
        cfg = model.native_config()
        params, keep = N.build_params(zip(slots, tensors), dev)
        need = C.c_size_t(0)
        N.check(getattr(N, entry.WORKSPACE_BYTES)(C.byref(cfg), B, T, C.byref(need)), entry.WORKSPACE_BYTES)
        ws = torch.empty(need.value + 256, dtype=torch.uint8, device=dev)  # owned by this node until backward
        shape = (B, model.n_sources, Cin, T) if entry.multichannel else (B, model.n_sources, T)
        out = torch.empty(shape, dtype=torch.float32, device=dev)
        N.check(getattr(N, entry.FWD)(C.byref(cfg), C.byref(params), x.data_ptr(), B, T, out.data_ptr(), *N.aligned(ws),
                                      N.stream_ptr(dev)), entry.FWD)
        model.last_launches = N.ctn_last_launch_count()
        # x and the parameters go through save_for_backward: an in-place update between forward and backward is detected by autograd
        # (version counters) instead of silently changing the weights the backward kernels see
        ctx.save_for_backward(x, *[t for t in tensors if t is not None])
        ctx.present = [t is not None for t in tensors]
        ctx.entry, ctx.cfg, ctx.ws, ctx.slots, ctx.model = entry, cfg, ws, slots, model
        return out

    @staticmethod
    def backward(ctx, d_out):
        if ctx.ws is None:
            raise RuntimeError("training node: backward was already run on this graph; the saved activations are released after the "
                               "first backward (retain_graph is not supported by the native training path)")
        saved = list(ctx.saved_tensors)
        x, it = saved[0], iter(saved[1:])
        tensors = tuple(next(it) if pres else None for pres in ctx.present)
        entry, ws, cfg = ctx.entry, ctx.ws, ctx.cfg
        dev = x.device
        B, _, T = x.shape
        d_out = d_out.contiguous()
        N.require_cuda(d_out)
        params, keep = N.build_params(zip(ctx.slots, tensors), dev)
        # one flat zero-initialised gradient buffer; every tensor starts 64-float aligned
        offs, total = [], 0
        for t in tensors:
            offs.append(total)
            total += 0 if t is None else (t.numel() + 63) // 64 * 64
        flat = torch.zeros(total, dtype=torch.float32, device=dev)
        gviews = [None if t is None else flat[o:o + t.numel()].view(t.shape) for t, o in zip(tensors, offs)]
        grads, keep2 = N.build_params(zip(ctx.slots, gviews), dev)
        d_x = None
        if entry.mixture_grad:
            d_x = torch.empty_like(x) if ctx.needs_input_grad[2] else None  # null: no gradient, no launch
            N.check(getattr(N, entry.BWD)(C.byref(cfg), C.byref(params), C.byref(grads), x.data_ptr(), d_out.data_ptr(), N.ptr(d_x), B,
                                          T, *N.aligned(ws), N.stream_ptr(dev)), entry.BWD)
        else:
            N.check(getattr(N, entry.BWD)(C.byref(cfg), C.byref(params), C.byref(grads), x.data_ptr(), d_out.data_ptr(), B, T,
                                          *N.aligned(ws), N.stream_ptr(dev)), entry.BWD)
        ctx.model.last_bwd_launches = N.ctn_last_launch_count()
        ctx.ws = None
        if entry.mixture_grad:
            # a node that ran earlier in this backward pass (a later fine-tune stage) owns the bucket: its views are what autograd
            # accumulates into the parameters' .grad, so add into them and pass nothing for the parameters
            task = torch._C._current_graph_task_id()
            owner = getattr(ctx.model, "_flat_grad_task", None)
            prev = getattr(ctx.model, "last_flat_grad", None)
            if task >= 0 and owner == (task, total) and prev is not None and prev.device == flat.device:
                prev.add_(flat)
                return (None, None, d_x) + (None,) * len(tensors)
            ctx.model._flat_grad_task = (task, total)
        ctx.model.last_flat_grad = flat
        return (None, None, d_x) + tuple(g if (t is not None and t.requires_grad) else None for g, t in zip(gviews, tensors))


def run_train(model, x, entry):
    """model(x) as one autograd node over the training step `entry` (train_entry(model)); x (B, Cin, T) on the device."""
    if x.requires_grad and not entry.mixture_grad:
        raise NotImplementedError("gradient w.r.t. the mixture is not built (the native backward stops at the encoder weights)")
    return TrainFn.apply(entry, model, x, *[t for _, t in param_list(model)])
