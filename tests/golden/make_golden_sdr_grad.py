"""Mints tests/golden/sdr_grad.pt from the UNMODIFIED reference on the CPU, the SDR criterion the WHAM and MUSDB18 recipes train with
(src/criterion/sdr.py:6-110 NegSDR, src/criterion/pit.py:9-77 PIT1d), in the reference's fp32 and from the same modules in fp64:
  * "pit": PIT1d(NegSDR(), S) on seeded (B, S, T) estimates and targets for S = 2 and 3: loss, pattern, loss per sample and the
    gradient of the batch mean w.r.t. the estimate;
  * "musdb": NegSDR() on a (B, S, C, T) batch standardised the way the MUSDB18 trainer does it (mixture mean and std over time,
    egs/musdb18/conv-tasnet/src/adhoc_driver.py:32-36), with its gradient w.r.t. the estimate;
  * "model": the tiny gLN Conv-TasNet's loss.backward() under PIT1d(NegSDR()), every parameter gradient kept, in the record
    layout of make_golden.grad_case.
Run from this directory's make_golden environment:
    python tests/golden/make_golden_sdr_grad.py"""
import os

import torch

import make_golden as MG
from criterion.sdr import NegSDR  # noqa: E402  (reference)
from criterion.pit import PIT1d  # noqa: E402  (reference)

TINY = dict(n_basis=16, kernel_size=4, sep_hidden_channels=16, sep_bottleneck_channels=8, sep_skip_channels=8, sep_num_blocks=2,
            sep_num_layers=3, causal=False, n_sources=2)
EPS = 1e-12  # the MUSDB18 trainer's standardisation epsilon


def pit_case(S, B=4, T=401, seed=0):
    g = torch.Generator().manual_seed(700 + S + seed)
    target = torch.randn(B, S, T, generator=g)
    est = target[:, torch.randperm(S, generator=g)] + 0.5 * torch.randn(B, S, T, generator=g)
    rec = {"input": est, "target": target}
    for dtype, sfx in ((torch.float32, ""), (torch.float64, "64")):
        x = est.to(dtype).clone().requires_grad_(True)
        crit = PIT1d(NegSDR(), S)
        loss, pattern = crit(x, target.to(dtype))
        loss.backward()
        loss_b, pattern_b = crit(x.detach(), target.to(dtype), batch_mean=False)
        assert torch.equal(pattern, pattern_b)
        rec.update({"loss" + sfx: loss.detach(), "pattern" + sfx: pattern, "loss_b" + sfx: loss_b.detach(), "grad" + sfx: x.grad})
    assert torch.equal(rec["pattern"], rec["pattern64"])
    return rec


def musdb_case(B=2, S=4, C=2, T=333, seed=41):
    g = torch.Generator().manual_seed(seed)
    sources = 0.2 * torch.randn(B, S, C, T, generator=g) + 0.05
    mixture = sources.sum(dim=1, keepdim=True)
    est = sources + 0.1 * torch.randn(B, S, C, T, generator=g)
    mean, std = mixture.mean(dim=-1, keepdim=True), mixture.std(dim=-1, keepdim=True)
    std_est, std_src = (est - mean) / (std + EPS), (sources - mean) / (std + EPS)
    rec = {"input": std_est, "target": std_src}
    for dtype, sfx in ((torch.float32, ""), (torch.float64, "64")):
        x = std_est.to(dtype).clone().requires_grad_(True)
        loss = NegSDR()(x, std_src.to(dtype))
        loss.backward()
        rec.update({"loss" + sfx: loss.detach(), "grad" + sfx: x.grad})
    return rec


def model_case(batch=2, T=203, wseed=11, xseed=21):
    cfg = MG.O.OracleConfig(**TINY)
    sd = MG.O.synth_state_dict(cfg, seed=wseed)
    mixture, sources = MG.O.synth_batch(batch, cfg.n_sources, T, seed=xseed)
    crit = PIT1d(NegSDR(), cfg.n_sources)

    def run(dtype):
        ref = MG.build_reference(cfg).to(dtype)
        ref.load_state_dict({k: v.to(dtype) for k, v in sd.items()}, strict=True)
        ref.train()
        out = ref(mixture.to(dtype))
        loss, perm = crit(out, sources.to(dtype))
        loss.backward()
        return ref, loss, perm

    ref, loss, perm = run(torch.float32)
    ref64, loss64, perm64 = run(torch.float64)
    assert torch.equal(perm, perm64)
    g64 = {k: p.grad.detach() for k, p in ref64.named_parameters()}
    grads = {}
    for k, p in ref.named_parameters():
        gr, d = p.grad.detach(), g64[k]
        grads[k] = {"sum": float(gr.double().sum()), "absmax": float(gr.abs().max()), "sample": gr.flatten().clone(),
                    "shape": tuple(gr.shape), "sample64": d.flatten().clone(), "sum64": float(d.sum()),
                    "absmax64": float(d.abs().max()), "fp32_vs_fp64_maxabs": float((gr.double() - d).abs().max())}
    return {"cfg": cfg.to_dict(), "batch": batch, "T": T, "wseed": wseed, "xseed": xseed, "stride": 1, "loss": loss.detach(),
            "loss64": float(loss64), "perm": perm, "grads": grads}


if __name__ == "__main__":
    rec = {"pit": {S: pit_case(S) for S in (2, 3)}, "musdb": musdb_case(), "model": model_case()}
    path = os.path.join(MG.HERE, "sdr_grad.pt")
    torch.save(rec, path)
    print("sdr_grad: PIT losses {} / MUSDB18 loss {:.6f} / model loss {:.6f} perm {} -> {} B".format(
        {S: round(float(r["loss"]), 6) for S, r in rec["pit"].items()}, float(rec["musdb"]["loss"]), float(rec["model"]["loss"]),
        rec["model"]["perm"].tolist(), os.path.getsize(path)))
