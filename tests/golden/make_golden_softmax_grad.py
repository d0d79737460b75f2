"""Mints tests/golden/tiny_softmax_grad.pt from the UNMODIFIED reference on the CPU: a small ConvTasNet(mask_nonlinear='softmax')
(the ORPIT and Sinkhorn PIT recipes, egs/wsj0-mix/orpit_conv-tasnet and egs/tutorials/{orpit,sinkpit}_conv-tasnet), in the
reference's fp32 and from the same modules in fp64 (the fp32 gradients are kept as their distance to fp64 only):
  * "orpit": the model's output, the ORPIT(NegSISDR()) loss over a PackedSequence of 2- and 3-speaker targets, its indices and
    every parameter gradient of ``loss.backward()`` (train.sh);
  * "finetune": the recursive fine-tune step on 3-speaker targets (finetune.sh; adhoc_driver.py, FinetuneTrainer): two stages of
    ``est = model(mixture); loss += ORPIT(est, sources); mixture = est[:, 1:]`` with the targets the first stage picked removed,
    then one backward, so the second stage's gradient flows through the first stage's estimate (the mixture gradient);
  * "sinkpit": an n_sources = 5 model under SinkPIT(NegSISDR(), n_sources=5) (egs/tutorials/sinkpit_conv-tasnet).
Every element is kept.  Run from this directory's make_golden environment:
    python tests/golden/make_golden_softmax_grad.py"""
import os

import torch
from torch.nn.utils.rnn import pack_sequence

import make_golden as MG
from criterion.pit import ORPIT, SinkPIT  # noqa: E402  (reference)
from criterion.sdr import NegSISDR  # noqa: E402  (reference)

TINY = dict(n_basis=16, kernel_size=4, sep_hidden_channels=16, sep_bottleneck_channels=8, sep_skip_channels=8, sep_num_blocks=2,
            sep_num_layers=3, causal=False, mask_nonlinear="softmax")
T = 203


def finetune_loss(model, mixture, sources, crit):
    """the fine-tune step's loss: n - 1 stages for n-speaker targets; each stage's 'rest' estimate is the next stage's mixture"""
    n = sources.size(1)
    total = 0
    for stage in range(n - 1):
        est = model(mixture)
        loss, idx = crit(est, sources)
        total = total + loss
        keep = [[j for j in range(n - stage) if j != int(idx[b])] for b in range(sources.size(0))]
        sources = torch.stack([sources[b, keep[b]] for b in range(sources.size(0))])
        mixture = est[:, 1:]
    return total


def _run(cfg, sd, dtype, fn):
    ref = MG.build_reference(cfg).to(dtype)
    assert [(k, tuple(v.shape)) for k, v in ref.state_dict().items()] == [(k, tuple(s)) for k, s in MG.O.state_dict_spec(cfg)]
    ref.load_state_dict({k: v.to(dtype) for k, v in sd.items()}, strict=True)
    ref.train()
    out, loss, extra = fn(ref, dtype)
    loss.backward()
    return out.detach(), loss.detach(), extra, {k: p.grad.detach().clone() for k, p in ref.named_parameters()}


def case(cfg, wseed, fn):
    sd = MG.O.synth_state_dict(cfg, seed=wseed)
    out, loss, extra, grads = _run(cfg, sd, torch.float32, fn)
    out64, loss64, extra64, grads64 = _run(cfg, sd, torch.float64, fn)
    return {"cfg": cfg.to_dict(), "wseed": wseed, "out": out, "out64": out64, "loss": float(loss), "loss64": float(loss64),
            "extra": extra, "extra64": extra64, "grads64": grads64,
            "fp32_vs_fp64_maxabs": {k: float((grads[k].double() - grads64[k]).abs().max()) for k in grads}}


def main():
    g = torch.Generator().manual_seed(35)
    rec = {}
    # ORPIT over a PackedSequence of 2- and 3-speaker targets; the mixture is the sum of each sample's targets
    lens = [2, 3, 3]
    tgts = [0.3 * torch.randn(n, T, generator=g) for n in lens]
    mixture = torch.stack([t.sum(dim=0, keepdim=True) for t in tgts])
    cfg = MG.O.OracleConfig(**TINY, n_sources=2)

    def orpit(ref, dtype):
        est = ref(mixture.to(dtype))
        loss, idx = ORPIT(NegSISDR())(est, pack_sequence([t.to(dtype) for t in tgts], enforce_sorted=False))
        return est, loss, idx

    rec["orpit"] = dict(case(cfg, 36, orpit), mixture=mixture, targets=tgts)
    # the two-stage fine-tune step on 3-speaker targets
    src3 = 0.3 * torch.randn(2, 3, T, generator=g)
    mix3 = src3.sum(dim=1, keepdim=True)

    def finetune(ref, dtype):
        est = ref(mix3.to(dtype))
        return est, finetune_loss(ref, mix3.to(dtype), src3.to(dtype), ORPIT(NegSISDR())), None

    rec["finetune"] = dict(case(cfg, 37, finetune), mixture=mix3, sources=src3)
    # SinkPIT with five outputs
    cfg5 = MG.O.OracleConfig(**TINY, n_sources=5)
    src5 = 0.3 * torch.randn(2, 5, T, generator=g)
    mix5 = src5.sum(dim=1, keepdim=True)

    def sink(ref, dtype):
        est = ref(mix5.to(dtype))
        loss, pattern = SinkPIT(NegSISDR(), n_sources=5)(est, src5.to(dtype))
        return est, loss, pattern

    rec["sinkpit"] = dict(case(cfg5, 38, sink), mixture=mix5, sources=src5)
    path = os.path.join(MG.HERE, "tiny_softmax_grad.pt")
    torch.save(rec, path)
    for k, r in rec.items():
        print("{}: out {} loss {:.6f} (fp64 {:.6f}), {} gradient tensors".format(k, tuple(r["out"].shape), r["loss"], r["loss64"],
                                                                                len(r["grads64"])))
    print("-> {} B".format(os.path.getsize(path)))


if __name__ == "__main__":
    main()
