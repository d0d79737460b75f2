"""Online (chunk-by-chunk) inference of a causal ConvTasNet or LSTM-TasNet: ``model.online(batch_size, max_chunk)``.

B streams advance together, one ``push`` per chunk (csrc/ctn_online.cu; csrc/ctn_tasnet.cu for LSTM-TasNet).  Each push of n samples returns n samples per
source, ``delay`` = kernel_size - stride samples late: with x everything pushed since the last reset, Y the concatenated
push outputs and Z = ``flush()``, ``Y[..., :delay]`` is zero and ``cat(Y[..., delay:], Z)`` equals ``model(x)``.

The state lives in one device buffer: the sample counter, the running cLN sums, each residual block's depthwise history, the
filter-bank carries, the weight images of every contraction (built here, once) and one chunk's scratch.  A push reads its
counters from the device, so a push captured in a CUDA graph replays correctly.  The weights must not change after
``online()``: every push compares the parameters' versions and raises if one did.

Envelope: causal=True (cLN; gLN needs the whole utterance), in_channels == 1, trainable bases, sigmoid or softmax mask, every
math mode.  Anything else raises NotImplementedError.

``TasOnlineSeparator`` is the same host logic over the ctn_tas_online_* entries: the state then carries the encoder's input, the
decoder's history and (h, c) of every LSTM layer (DESIGN.md section 18).  Envelope: causal=True (a non-causal model is
bidirectional), enc_basis='trainable' (the gated encoder divides by the norm of the whole signal), rnn_type='lstm', in_channels
== 1, sigmoid or softmax mask, a hidden size inside the recurrence kernel's envelope, every math mode.
"""
import ctypes as C

import torch

from .. import _native as N


class OnlineSeparator:
    # ctn_online_state_bytes / _init / _reset / _push / _flush of the model's family
    ENTRIES = ("ctn_online_state_bytes", "ctn_online_init", "ctn_online_reset", "ctn_online_push", "ctn_online_flush")

    @staticmethod
    def check_model(model):
        """NotImplementedError for a model outside the envelope (before any CUDA call)"""
        if not model.causal:
            raise NotImplementedError("online inference needs a causal model (cLN): gLN statistics span the whole utterance")
        if model.in_channels != 1:
            raise NotImplementedError("online inference is monaural (in_channels == 1)")
        if model.enc_basis != "trainable" or model.dec_basis != "trainable":
            raise NotImplementedError("online inference needs trainable filter banks")

    def native(self, model):
        """-> (config, parameters, keep) of the C entries; keep must outlive the state"""
        params, keep = model.native_params(self.device)
        return model.native_config(), params, keep

    def __init__(self, model, batch_size=1, max_chunk=256):
        self.check_model(model)
        if batch_size <= 0:
            raise ValueError("batch_size must be positive, got {}".format(batch_size))
        if max_chunk <= 0 or max_chunk % model.stride != 0:
            raise ValueError("max_chunk must be a positive multiple of the stride ({}), got {}".format(model.stride, max_chunk))
        self.model = model
        self.batch_size, self.max_chunk = int(batch_size), int(max_chunk)
        self.stride, self.kernel_size, self.n_sources = model.stride, model.kernel_size, model.n_sources
        self.delay = model.kernel_size - model.stride
        self.device = model.encoder.conv1d.weight.device
        if self.device.type != "cuda":
            raise RuntimeError("ctn_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        self._state_bytes, self._init, self._reset, self._push, self._flush = [getattr(N, e) for e in self.ENTRIES]
        self._cfg, self._params, self._keep = self.native(model)
        self._watch = list(model.parameters())
        self._versions = [(p.data_ptr(), p._version) for p in self._watch]
        need = C.c_size_t(0)
        N.check(self._state_bytes(C.byref(self._cfg), self.batch_size, self.max_chunk // self.stride, C.byref(need)), self.ENTRIES[0])
        self.state_bytes = need.value
        self._state = torch.empty(need.value + 256, dtype=torch.uint8, device=self.device)
        self._base, _ = N.aligned(self._state)
        with torch.cuda.device(self.device):
            N.check(self._init(C.byref(self._cfg), C.byref(self._params), self.batch_size, self.max_chunk // self.stride, self._base,
                               need.value, N.stream_ptr(self.device)), self.ENTRIES[1])
        self._flushed = False
        self.last_launches = 0

    def _check_weights(self):
        if [(p.data_ptr(), p._version) for p in self._watch] != self._versions:
            raise RuntimeError("a weight of the model changed after online(): its images are stale; call model.online() again")

    def push(self, x):
        """x (batch_size, 1, n) float32 CUDA, n a multiple of the stride, 0 < n <= max_chunk -> y (batch_size, n_sources, n)"""
        if self._flushed:
            raise RuntimeError("push after flush(): call reset() first")
        if x.dim() != 3 or x.size(0) != self.batch_size or x.size(1) != 1:
            raise ValueError("x.size() is expected ({}, 1, n), but given {}".format(self.batch_size, tuple(x.size())))
        n = x.size(2)
        if n <= 0 or n % self.stride != 0 or n > self.max_chunk:
            raise ValueError("a push takes a positive multiple of the stride ({}) up to max_chunk = {} samples, got {}".format(
                self.stride, self.max_chunk, n))
        if N.require_cuda(x) != self.device:
            raise RuntimeError("x must live on {}".format(self.device))
        self._check_weights()
        x = x.contiguous()
        y = torch.empty(self.batch_size, self.n_sources, n, dtype=torch.float32, device=self.device)
        with torch.no_grad(), torch.cuda.device(self.device):
            N.check(self._push(C.byref(self._cfg), C.byref(self._params), self._base, x.data_ptr(), self.batch_size,
                               self.max_chunk // self.stride, n, y.data_ptr(), N.stream_ptr(self.device)), self.ENTRIES[3])
        self.last_launches = N.ctn_last_launch_count()
        return y

    def flush(self):
        """-> (batch_size, n_sources, delay): the last `delay` samples of the offline output.  ValueError when fewer than
        kernel_size samples were pushed since the reset.  Synchronises the stream once (it reads the sample count)."""
        y = torch.empty(self.batch_size, self.n_sources, self.delay, dtype=torch.float32, device=self.device)
        with torch.no_grad(), torch.cuda.device(self.device):
            N.check(self._flush(C.byref(self._cfg), self._base, self.batch_size, y.data_ptr(), N.stream_ptr(self.device)),
                    self.ENTRIES[4])
        self._flushed = True
        return y

    def reset(self):
        """zero history, zero statistics, zero samples; the weight images are kept"""
        with torch.cuda.device(self.device):
            N.check(self._reset(C.byref(self._cfg), self._base, self.batch_size, N.stream_ptr(self.device)), self.ENTRIES[2])
        self._flushed = False


class TasOnlineSeparator(OnlineSeparator):
    """online inference of a causal LSTM-TasNet (models.tasnet.TasNet): the contract of OnlineSeparator"""
    ENTRIES = ("ctn_tas_online_state_bytes", "ctn_tas_online_init", "ctn_tas_online_reset", "ctn_tas_online_push",
               "ctn_tas_online_flush")

    @staticmethod
    def check_model(model):
        if model.enc_basis == "trainableGated":
            raise NotImplementedError("online inference needs enc_basis='trainable': the gated encoder divides each signal by its L2 "
                                      "norm over the whole signal, which no stream knows before it ends")
        if not model.causal:
            raise NotImplementedError("online inference needs a causal model: causal=False runs bidirectional LSTMs, whose reverse "
                                      "pass starts at the end of the signal")
        if model.in_channels != 1:
            raise NotImplementedError("online inference is monaural (in_channels == 1)")
        model.separator.check_envelope()  # rnn_type 'lstm', sigmoid or softmax mask

    def native(self, model):
        from .tdcn import resolve_math
        from . import tdcn as _tdcn
        sep = model.separator
        sep.check_hidden()
        cfg = N.TasConfig(n_basis=model.n_basis, kernel_size=model.kernel_size, stride=model.stride, hidden=sep.hidden_channels,
                          num_blocks=sep.num_blocks, num_layers=sep.num_layers, n_sources=model.n_sources, causal=int(model.causal),
                          gated=0, enc_relu=int(model.encoder.nonlinear), mask_softmax=int(sep.mask_softmax),
                          math=resolve_math(model.math if model.math is not None else _tdcn.DEFAULT_MATH), eps=float(sep.eps))
        keep = []

        def dev_ptr(t):
            if t.device != self.device or t.dtype != torch.float32:
                raise RuntimeError("parameters must be float32 on {}".format(self.device))
            if not t.is_contiguous():
                t = t.contiguous()
                keep.append(t)
            return t.data_ptr()

        lstm = []
        for rnn in sep.rnn:
            for k in range(sep.num_layers):
                lstm += [dev_ptr(getattr(rnn, n + "_l{}".format(k))) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
        arr = (N._fp * len(lstm))(*lstm)
        keep.append(arr)
        params = N.TasParams(enc_w=dev_ptr(model.encoder.conv1d.weight), gamma=dev_ptr(sep.gamma), beta=dev_ptr(sep.beta),
                             lstm=C.cast(arr, C.POINTER(N._fp)), fc_w=dev_ptr(sep.fc.weight), fc_b=dev_ptr(sep.fc.bias),
                             dec_w=dev_ptr(model.decoder.conv_transpose1d.weight))
        return cfg, params, keep
