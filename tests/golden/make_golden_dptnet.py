#!/usr/bin/env python
"""Mint DPTNet golden vectors from the UNMODIFIED reference (run where the reference's src/ is available).

    python tests/golden/make_golden_dptnet.py          # writes tests/golden/dptnet.pt

The reference's DPTNet is built as-is, loaded with seeded weights from tests/dptnet_ref.py (``synth_state_dict``) through
``load_state_dict(strict=True)`` and run in fp32 on the CPU in eval mode.  Stored per case: the config, the seed, the
reference's module names and state_dict keys, the input and the output.  Weights are not stored: they are regenerated from
the seed.
"""
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("DPTNET_REF_SRC", "/root/reference/src")
sys.path.insert(0, REF_SRC)
sys.path.insert(0, os.path.dirname(HERE))
warnings.simplefilter("ignore")
from models.dptnet import DPTNet  # noqa: E402  (reference)

import dptnet_ref as R  # noqa: E402

CASES = {
    "tiny": dict(n_basis=32, kernel_size=4, stride=2, enc_nonlinear="relu", sep_bottleneck_channels=32, sep_hidden_channels=32,
                 sep_chunk_size=16, sep_hop_size=8, sep_num_blocks=2, sep_num_heads=4, mask_nonlinear="sigmoid", n_sources=2,
                 eps=1e-12, batch=2, T=301, seed=11),
    "recipe_2spk": dict(n_basis=64, kernel_size=2, stride=1, enc_nonlinear="relu", sep_bottleneck_channels=64, sep_hidden_channels=128,
                        sep_chunk_size=250, sep_hop_size=125, sep_num_blocks=6, sep_num_heads=4, mask_nonlinear="relu", n_sources=2,
                        eps=1e-12, batch=1, T=800, seed=12),
    "recipe_3spk": dict(n_basis=64, kernel_size=2, stride=1, enc_nonlinear="relu", sep_bottleneck_channels=64, sep_hidden_channels=128,
                        sep_chunk_size=250, sep_hop_size=125, sep_num_blocks=6, sep_num_heads=4, mask_nonlinear="relu", n_sources=3,
                        eps=1e-12, batch=2, T=700, seed=13),
}


def build(cfg):
    return DPTNet(cfg["n_basis"], cfg["kernel_size"], stride=cfg["stride"], enc_basis="trainable", dec_basis="trainable",
                  enc_nonlinear=cfg["enc_nonlinear"], sep_bottleneck_channels=cfg["sep_bottleneck_channels"],
                  sep_hidden_channels=cfg["sep_hidden_channels"], sep_chunk_size=cfg["sep_chunk_size"], sep_hop_size=cfg["sep_hop_size"],
                  sep_num_blocks=cfg["sep_num_blocks"], sep_num_heads=cfg["sep_num_heads"], mask_nonlinear=cfg["mask_nonlinear"],
                  causal=False, n_sources=cfg["n_sources"], eps=cfg["eps"])


def main():
    torch.set_num_threads(8)
    out = {}
    for name, cfg in CASES.items():
        model = build(cfg).eval()
        keys_shapes = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
        model.load_state_dict(R.synth_state_dict(keys_shapes, cfg["seed"]), strict=True)
        g = torch.Generator().manual_seed(cfg["seed"] + 1000)
        x = torch.randn(cfg["batch"], 1, cfg["T"], generator=g)
        with torch.no_grad():
            y = model(x)
        out[name] = {"cfg": cfg, "keys_shapes": keys_shapes, "modules": [(n, type(m).__name__) for n, m in model.named_modules()],
                     "x": x, "out": y}
        print(name, tuple(y.shape), float(y.abs().max()))
    torch.save(out, os.path.join(HERE, "dptnet.pt"))


if __name__ == "__main__":
    main()
