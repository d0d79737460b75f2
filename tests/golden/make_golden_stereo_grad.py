"""Mints tests/golden/tiny_stereo_grad.pt from the UNMODIFIED reference on the CPU: a small ConvTasNet(in_channels=2) (the 4-D
input (B, 1, 2, T) of the MUSDB18 recipes), its output, the recipe's loss MeanSquaredError(dim=-1, reduction='mean') and every
parameter gradient of ``loss.backward()``, in the reference's fp32 and from the same modules in fp64; plus the reference's
MeanSquaredError / MeanAbsoluteError (src/criterion/distance.py) over the dim / reduction / batch_mean combinations on seeded
inputs.  Every element is kept.  Run from this directory's make_golden environment:
    python tests/golden/make_golden_stereo_grad.py"""
import os

import torch

import make_golden as MG
from criterion.distance import MeanAbsoluteError, MeanSquaredError  # noqa: E402  (reference)

CFG = dict(n_basis=16, kernel_size=4, sep_hidden_channels=16, sep_bottleneck_channels=8, sep_skip_channels=8, sep_num_blocks=2,
           sep_num_layers=3, causal=False, n_sources=3, in_channels=2)
DIMS = [-1, 1, 2, (1, 2), (2, 3), (1, 2, 3)]
REDUCTIONS = [None, "mean", "sum"]


def model_grad(batch=2, T=203, wseed=15, xseed=25):
    cfg = MG.O.OracleConfig(**CFG)
    sd = MG.O.synth_state_dict(cfg, seed=wseed)
    g = torch.Generator().manual_seed(xseed)
    mixture = 0.3 * torch.randn(batch, 1, cfg.in_channels, T, generator=g)
    sources = 0.3 * torch.randn(batch, cfg.n_sources, cfg.in_channels, T, generator=g)
    crit = MeanSquaredError(dim=-1, reduction="mean")

    def run(dtype):
        ref = MG.build_reference(cfg).to(dtype)
        assert [(k, tuple(v.shape)) for k, v in ref.state_dict().items()] == [(k, tuple(s)) for k, s in MG.O.state_dict_spec(cfg)]
        ref.load_state_dict({k: v.to(dtype) for k, v in sd.items()}, strict=True)
        ref.train()
        out = ref(mixture.to(dtype))
        loss = crit(out, sources.to(dtype))
        loss.backward()
        return out.detach(), loss.detach(), {k: p.grad.detach().clone() for k, p in ref.named_parameters()}

    out, loss, grads = run(torch.float32)
    out64, loss64, grads64 = run(torch.float64)
    return {"cfg": cfg.to_dict(), "wseed": wseed, "mixture": mixture, "sources": sources, "out": out, "out64": out64,
            "loss": loss, "loss64": float(loss64), "grads": grads, "grads64": grads64,
            "fp32_vs_fp64_maxabs": {k: float((grads[k].double() - grads64[k]).abs().max()) for k in grads}}


def criteria():
    g = torch.Generator().manual_seed(26)
    est = torch.randn(3, 4, 2, 37, generator=g)
    tgt = torch.randn(3, 4, 2, 37, generator=g)
    rec = {"input": est, "target": tgt}
    for name, cls in (("mse", MeanSquaredError), ("mae", MeanAbsoluteError)):
        for dim in DIMS:
            for red in REDUCTIONS:
                for bm in (True, False):
                    rec[(name, dim, red, bm)] = cls(dim=dim, reduction=red)(est, tgt, batch_mean=bm)
    return rec


if __name__ == "__main__":
    rec = model_grad()
    rec["criteria"] = criteria()
    path = os.path.join(MG.HERE, "tiny_stereo_grad.pt")
    torch.save(rec, path)
    print("tiny_stereo_grad: out {} loss {:.6f}, {} gradient tensors, {} criterion values -> {} B".format(
        tuple(rec["out"].shape), float(rec["loss"]), len(rec["grads"]), len(rec["criteria"]) - 2, os.path.getsize(path)))
