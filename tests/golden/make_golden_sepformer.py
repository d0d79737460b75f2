#!/usr/bin/env python
"""Mint SepFormer golden vectors from the UNMODIFIED reference (run where the reference's src/ is available).

    python tests/golden/make_golden_sepformer.py          # writes tests/golden/sepformer.pt

The reference's SepFormer is built as-is, loaded with seeded weights from tests/sepformer_ref.py (``synth_state_dict``, which
keeps the positional-encoding buffers the reference builds) through ``load_state_dict(strict=True)`` and run in fp32 on the CPU
in eval mode.  Stored per case: the config, the seed, the reference's module names and state_dict keys, the input and the
output, and the reference's own ``get_config()`` (the checkpoint header its trainer writes).  Weights are not stored: they are regenerated from the seed.
"""
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("SEPFORMER_REF_SRC", "/root/reference/src")
sys.path.insert(0, REF_SRC)
sys.path.insert(0, os.path.dirname(HERE))
warnings.simplefilter("ignore")
from models.sepformer import SepFormer  # noqa: E402  (reference)

import sepformer_ref as R  # noqa: E402

RECIPE = dict(n_basis=256, kernel_size=16, stride=8, enc_nonlinear="relu", sep_bottleneck_channels=256, sep_chunk_size=250,
              sep_hop_size=125, sep_num_blocks=2, sep_num_layers_intra=8, sep_num_layers_inter=8, sep_num_heads_intra=8,
              sep_num_heads_inter=8, sep_d_ff_intra=1024, sep_d_ff_inter=1024, mask_nonlinear="relu", eps=1e-12)
CASES = {
    "tiny": dict(n_basis=32, kernel_size=16, stride=8, enc_nonlinear="relu", sep_bottleneck_channels=32, sep_chunk_size=16,
                 sep_hop_size=8, sep_num_blocks=2, sep_num_layers_intra=2, sep_num_layers_inter=2, sep_num_heads_intra=4,
                 sep_num_heads_inter=4, sep_d_ff_intra=64, sep_d_ff_inter=64, mask_nonlinear="sigmoid", eps=1e-12, n_sources=2,
                 batch=2, T=1203, seed=21),
    "recipe_2spk": dict(RECIPE, n_sources=2, batch=1, T=8000, seed=22),
    "recipe_3spk": dict(RECIPE, n_sources=3, batch=2, T=4000, seed=23),
}


def build(cfg):
    return SepFormer(cfg["n_basis"], cfg["kernel_size"], stride=cfg["stride"], enc_basis="trainable", dec_basis="trainable",
                     enc_nonlinear=cfg["enc_nonlinear"], sep_bottleneck_channels=cfg["sep_bottleneck_channels"],
                     sep_chunk_size=cfg["sep_chunk_size"], sep_hop_size=cfg["sep_hop_size"], sep_num_blocks=cfg["sep_num_blocks"],
                     sep_num_layers_intra=cfg["sep_num_layers_intra"], sep_num_layers_inter=cfg["sep_num_layers_inter"],
                     sep_num_heads_intra=cfg["sep_num_heads_intra"], sep_num_heads_inter=cfg["sep_num_heads_inter"],
                     sep_d_ff_intra=cfg["sep_d_ff_intra"], sep_d_ff_inter=cfg["sep_d_ff_inter"], mask_nonlinear=cfg["mask_nonlinear"],
                     causal=False, n_sources=cfg["n_sources"], eps=cfg["eps"])


def main():
    torch.set_num_threads(8)
    out = {}
    for name, cfg in CASES.items():
        model = build(cfg).eval()
        keys_shapes = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
        sd = R.synth_state_dict(keys_shapes, cfg["seed"])
        for k, v in model.state_dict().items():  # the buffers the reference built are the ones the seeded dict carries
            if k.endswith(R.PE_KEY):
                assert torch.equal(v, sd[k]), k
        model.load_state_dict(sd, strict=True)
        g = torch.Generator().manual_seed(cfg["seed"] + 1000)
        x = torch.randn(cfg["batch"], 1, cfg["T"], generator=g)
        with torch.no_grad():
            y = model(x)
        out[name] = {"cfg": cfg, "keys_shapes": keys_shapes, "modules": [(n, type(m).__name__) for n, m in model.named_modules()],
                     "ref_config": model.get_config(), "x": x, "out": y}
        print(name, tuple(y.shape), float(y.abs().max()))
    torch.save(out, os.path.join(HERE, "sepformer.pt"))


if __name__ == "__main__":
    main()
