"""Native training-step remainder (SURVEY.md 8f-3): global-norm gradient clipping + Adam on the flat gradient bucket.

Replaces ``torch.nn.utils.clip_grad_norm_(model.parameters(), max_norm)`` + ``torch.optim.Adam.step()`` of the reference
trainer (egs/wsj0-mix/common/src/driver.py:149-157) with ONE C call = 3 kernel launches over the flat bucket the native backward
fills (ctn_b200/models/_train.py): sum of squares -> clip coefficient + Adam update of every parameter tensor (chunk table) ->
step counter.  Step counter and learning rate live on the device (CUDA-graph replayable; ``set_lr`` implements the halving
scheduler of egs/wsj0-mix/conv-tasnet/src/adhoc_driver.py:25-39 without re-capture).  Same arithmetic as torch.optim.Adam
(amsgrad=False, maximize=False): parity to ~1e-7 is tested against it (tests/test_train_gpu.py)."""
import ctypes as C

import torch

from . import _native as N


class FlatClipAdam:
    def __init__(self, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, max_norm=None):
        self.model = model
        self.params = [p for p in model.parameters() if p.requires_grad]
        if not self.params:
            raise ValueError("no trainable parameters")
        dev = self.params[0].device
        if dev.type != "cuda":
            raise RuntimeError("ctn_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        self.dev, self.betas, self.eps, self.weight_decay = dev, betas, eps, weight_decay
        self.max_norm = 0.0 if max_norm is None else float(max_norm)
        self.lr = torch.full((1,), float(lr), dtype=torch.float32, device=dev)
        self.step_count = torch.zeros(1, dtype=torch.int64, device=dev)
        self.sumsq = torch.zeros(1, dtype=torch.float64, device=dev)
        self.total_norm = torch.zeros(1, dtype=torch.float32, device=dev)
        self._layout = None
        self.launches_per_step = 3

    def zero_grad(self, set_to_none=True):
        for p in self.params:
            p.grad = None

    def set_lr(self, lr):
        self.lr.fill_(float(lr))

    def _bind(self, flat):
        """(Re)build the device tables for the current flat bucket layout: every p.grad must be a view into `flat`."""
        offs, numel = [], []
        base, esz = flat.data_ptr(), flat.element_size()
        for p in self.params:
            g = p.grad
            if g is None or not g.is_contiguous() or not (base <= g.data_ptr() < base + flat.numel() * esz):
                raise RuntimeError("FlatClipAdam needs the gradients as views of model.last_flat_grad (native backward)")
            offs.append((g.data_ptr() - base) // esz)
            numel.append(p.numel())
        key = (flat.numel(), tuple(offs), tuple(p.data_ptr() for p in self.params))
        if self._layout is not None and self._layout["key"] == key:
            return self._layout
        n = len(self.params)
        numel_c = (C.c_int * n)(*numel)
        n_chunks = N.ctn_clip_adam_chunks(numel_c, n, None, None, 0)
        ct, co = (C.c_int * n_chunks)(), (C.c_int * n_chunks)()
        N.ctn_clip_adam_chunks(numel_c, n, ct, co, n_chunks)
        table = torch.tensor([[ct[i], co[i]] for i in range(n_chunks)], dtype=torch.int32).to(self.dev)
        lay = dict(key=key, n_chunks=n_chunks, table=table,
                   ptrs=torch.tensor([p.data_ptr() for p in self.params], dtype=torch.int64).to(self.dev),
                   offs=torch.tensor(offs, dtype=torch.int64).to(self.dev), numel=torch.tensor(numel, dtype=torch.int32).to(self.dev))
        if self._layout is None or self._layout["key"][0] != key[0] or self._layout["key"][1] != key[1]:
            lay["m"] = torch.zeros(flat.numel(), dtype=torch.float32, device=self.dev)
            lay["v"] = torch.zeros(flat.numel(), dtype=torch.float32, device=self.dev)
        else:
            lay["m"], lay["v"] = self._layout["m"], self._layout["v"]
        self._layout = lay
        return lay

    def step(self):
        flat = getattr(self.model, "last_flat_grad", None)
        if flat is None:
            raise RuntimeError("FlatClipAdam.step() before a native backward (model.last_flat_grad is not set)")
        lay = self._bind(flat)
        with torch.cuda.device(self.dev):
            N.check(N.ctn_clip_adam_step(lay["table"].data_ptr(), lay["n_chunks"], lay["ptrs"].data_ptr(), lay["offs"].data_ptr(),
                                         lay["numel"].data_ptr(), len(self.params), flat.data_ptr(), flat.numel(), lay["m"].data_ptr(),
                                         lay["v"].data_ptr(), self.sumsq.data_ptr(), self.lr.data_ptr(), self.step_count.data_ptr(),
                                         float(self.betas[0]), float(self.betas[1]), float(self.eps), float(self.weight_decay),
                                         float(self.max_norm), self.total_norm.data_ptr(), N.stream_ptr(self.dev)), "ctn_clip_adam_step")
        return self.total_norm

    def state_dict(self):
        lay = self._layout
        return {"lr": float(self.lr[0]), "step": int(self.step_count[0]), "betas": self.betas, "eps": self.eps, "weight_decay": self.weight_decay,
                "max_norm": self.max_norm, "exp_avg": None if lay is None else lay["m"].clone(), "exp_avg_sq": None if lay is None else lay["v"].clone()}
