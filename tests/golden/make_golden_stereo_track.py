"""Mints tests/golden/tiny_stereo_track.pt from the UNMODIFIED reference on the CPU: a whole stereo "track" separated by a small
ConvTasNet(in_channels=2) (the tiny config of make_golden_stereo_grad.py) the way the MUSDB18 recipe's tester separates a track
(egs/musdb18/conv-tasnet, test.sh with its adhoc_dataset.py / adhoc_driver.py): zero-pad to a multiple of the segment, cut into
segments that share no samples, standardise every segment and channel on its own with (x - mean) / (std + 1e-12) (unbiased
std, the padded zeros included), one forward per segment, std * estimate + mean, concatenate, crop to T.  Those modules import
musdb, museval and torchaudio, so the steps are restated here.  The same steps also run on the cross-faded layout of
separate_long (chunks every `hop`, the last one ending at T, sin^2 / cos^2 ramps), which the recipe does not have.

Both routes run in the reference's fp32 and, from the same modules, in fp64.  The track holds an all-zero segment and a segment
with a large DC offset; T is not a multiple of the segment.  Run from this directory's make_golden environment:
    python tests/golden/make_golden_stereo_track.py"""
import math
import os

import torch

import make_golden as MG
from make_golden_stereo_grad import CFG

EPS = 1e-12
SEGMENT, HOP, T, BATCH = 128, 96, 709, 1


def mixture(seed=35):
    g = torch.Generator().manual_seed(seed)
    x = 0.3 * torch.randn(BATCH, 1, CFG["in_channels"], T, generator=g)
    x[0, :, :, SEGMENT:2 * SEGMENT] = 0.0                      # segment 1: silence in both channels
    x[0, :, 0, 3 * SEGMENT:4 * SEGMENT] += 40.0                # segment 3: a DC offset on the left channel
    x[0, :, 1, 3 * SEGMENT:4 * SEGMENT] -= 25.0                # ... and another on the right
    return x


def starts_of(hop):
    if hop is None:
        return [k * SEGMENT for k in range(-(-T // SEGMENT))]
    s, out = 0, []
    while s + SEGMENT < T:
        out.append(s)
        s += hop
    return out + [T - SEGMENT]


def ramps(starts):
    """(K, Tp) cross-fade weights: sin^2 rise over the samples shared with the previous chunk, cos^2 fall over those shared with
    the next, half-sample offsets"""
    Tp = starts[-1] + SEGMENT
    w = torch.zeros(len(starts), Tp, dtype=torch.float64)
    for k, s0 in enumerate(starts):
        wk = torch.ones(SEGMENT, dtype=torch.float64)
        if k > 0:
            a = starts[k - 1] + SEGMENT - s0
            r = torch.arange(a, dtype=torch.float64)
            wk[:a] *= torch.sin(math.pi / 2 * (r + 0.5) / a) ** 2
        if k + 1 < len(starts):
            n = s0 + SEGMENT - starts[k + 1]
            q = torch.arange(n, dtype=torch.float64)
            wk[SEGMENT - n:] *= torch.cos(math.pi / 2 * (q + 0.5) / n) ** 2
        w[k, s0:s0 + SEGMENT] = wk
    return w


def route(model, x, hop, dtype):
    """x (B, 1, C, T) -> dict of the steps' results in `dtype`"""
    starts = starts_of(hop)
    K, Tp = len(starts), starts[-1] + SEGMENT
    xp = torch.nn.functional.pad(x.to(dtype), (0, Tp - T))      # only the tester's layout reads past T
    seg = torch.stack([xp[..., s0:s0 + SEGMENT] for s0 in starts], dim=1)   # (B, K, 1, C, Lc)
    seg = seg.reshape(BATCH * K, 1, CFG["in_channels"], SEGMENT)
    mean, std = seg.mean(dim=-1, keepdim=True), seg.std(dim=-1, keepdim=True)
    z = (seg - mean) / (std + EPS)
    est = torch.cat([model(z[i:i + 1]) for i in range(BATCH * K)])           # (B K, S, C, Lc), one forward per segment
    y = std * est + mean
    S, Cn = est.shape[1], est.shape[2]
    y = y.reshape(BATCH, K, S, Cn, SEGMENT)
    if hop is None:
        out = y.permute(0, 2, 3, 1, 4).reshape(BATCH, S, Cn, K * SEGMENT)[..., :T]
    else:
        w = ramps(starts).to(dtype)
        num = torch.zeros(BATCH, S, Cn, Tp, dtype=dtype)
        for k, s0 in enumerate(starts):
            num[..., s0:s0 + SEGMENT] += w[k, s0:s0 + SEGMENT] * y[:, k]
        out = (num / w.sum(0))[..., :T]
    return {"starts": starts, "mean": mean.reshape(BATCH, K, Cn), "std": std.reshape(BATCH, K, Cn),
            "chunks": z.reshape(BATCH * K, Cn, SEGMENT), "est": est.detach(), "out": out.detach()}


def main():
    cfg = MG.O.OracleConfig(**CFG)
    wseed = 15
    sd = MG.O.synth_state_dict(cfg, seed=wseed)
    x = mixture()
    rec = {"cfg": cfg.to_dict(), "wseed": wseed, "mixture": x, "segment": SEGMENT, "hop": HOP, "eps": EPS}
    with torch.no_grad():
        for name, hop in (("tester", None), ("crossfaded", HOP)):
            r = {}
            for dtype, tag in ((torch.float32, ""), (torch.float64, "64")):
                ref = MG.build_reference(cfg).to(dtype)
                ref.load_state_dict({k: v.to(dtype) for k, v in sd.items()}, strict=True)
                ref.eval()
                for k, v in route(ref, x, hop, dtype).items():
                    if k == "chunks":                                     # the standardised inputs follow from mixture, mean, std
                        continue
                    if tag or k in ("starts", "mean", "std", "out"):      # the chunk estimates are kept in fp64 only
                        r[k + tag] = v.clone() if torch.is_tensor(v) else v
            r["fp32_vs_fp64_maxabs"] = float((r["out"].double() - r["out64"]).abs().max())
            rec[name] = r
    path = os.path.join(MG.HERE, "tiny_stereo_track.pt")
    torch.save(rec, path)
    for name in ("tester", "crossfaded"):
        r = rec[name]
        print("{}: {} segments, out {} fp32 vs fp64 {:.2e}".format(name, len(r["starts"]), tuple(r["out"].shape), r["fp32_vs_fp64_maxabs"]))
    print("-> {} B".format(os.path.getsize(path)))


if __name__ == "__main__":
    main()
