"""Online (chunk-by-chunk) inference of a causal ConvTasNet: ``model.online(batch_size, max_chunk)``.

B streams advance together, one ``push`` per chunk (csrc/ctn_online.cu).  Each push of n samples returns n samples per
source, ``delay`` = kernel_size - stride samples late: with x everything pushed since the last reset, Y the concatenated
push outputs and Z = ``flush()``, ``Y[..., :delay]`` is zero and ``cat(Y[..., delay:], Z)`` equals ``model(x)``.

The state lives in one device buffer: the sample counter, the running cLN sums, each residual block's depthwise history, the
filter-bank carries, the weight images of every contraction (built here, once) and one chunk's scratch.  A push reads its
counters from the device, so a push captured in a CUDA graph replays correctly.  The weights must not change after
``online()``: every push compares the parameters' versions and raises if one did.

Envelope: causal=True (cLN; gLN needs the whole utterance), in_channels == 1, trainable bases, sigmoid or softmax mask, every
math mode.  Anything else raises NotImplementedError.
"""
import ctypes as C

import torch

from .. import _native as N


class OnlineSeparator:
    def __init__(self, model, batch_size=1, max_chunk=256):
        if not model.causal:
            raise NotImplementedError("online inference needs a causal model (cLN): gLN statistics span the whole utterance")
        if model.in_channels != 1:
            raise NotImplementedError("online inference is monaural (in_channels == 1)")
        if model.enc_basis != "trainable" or model.dec_basis != "trainable":
            raise NotImplementedError("online inference needs trainable filter banks")
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
        self._cfg = model.native_config()
        self._params, self._keep = model.native_params(self.device)
        self._watch = list(model.parameters())
        self._versions = [(p.data_ptr(), p._version) for p in self._watch]
        need = C.c_size_t(0)
        N.check(N.ctn_online_state_bytes(C.byref(self._cfg), self.batch_size, self.max_chunk // self.stride, C.byref(need)),
                "ctn_online_state_bytes")
        self.state_bytes = need.value
        self._state = torch.empty(need.value + 256, dtype=torch.uint8, device=self.device)
        self._base, _ = N.aligned(self._state)
        with torch.cuda.device(self.device):
            N.check(N.ctn_online_init(C.byref(self._cfg), C.byref(self._params), self.batch_size, self.max_chunk // self.stride,
                                      self._base, need.value, N.stream_ptr(self.device)), "ctn_online_init")
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
            N.check(N.ctn_online_push(C.byref(self._cfg), C.byref(self._params), self._base, x.data_ptr(), self.batch_size,
                                      self.max_chunk // self.stride, n, y.data_ptr(), N.stream_ptr(self.device)), "ctn_online_push")
        self.last_launches = N.ctn_last_launch_count()
        return y

    def flush(self):
        """-> (batch_size, n_sources, delay): the last `delay` samples of the offline output.  ValueError when fewer than
        kernel_size samples were pushed since the reset.  Synchronises the stream once (it reads the sample count)."""
        y = torch.empty(self.batch_size, self.n_sources, self.delay, dtype=torch.float32, device=self.device)
        with torch.no_grad(), torch.cuda.device(self.device):
            N.check(N.ctn_online_flush(C.byref(self._cfg), self._base, self.batch_size, y.data_ptr(), N.stream_ptr(self.device)),
                    "ctn_online_flush")
        self._flushed = True
        return y

    def reset(self):
        """zero history, zero statistics, zero samples; the weight images are kept"""
        with torch.cuda.device(self.device):
            N.check(N.ctn_online_reset(C.byref(self._cfg), self._base, self.batch_size, N.stream_ptr(self.device)), "ctn_online_reset")
        self._flushed = False
