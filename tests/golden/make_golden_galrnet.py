#!/usr/bin/env python
"""Mint GALRNet golden vectors from the UNMODIFIED reference (run where the reference's src/ is available).

    python tests/golden/make_golden_galrnet.py          # writes tests/golden/galrnet.pt

The reference's GALRNet is built as-is, loaded with seeded weights from tests/galrnet_ref.py (``synth_state_dict``) through
``load_state_dict(strict=True)`` and run in fp32 on the CPU in eval mode.  Stored per case: the config, the seed, the
reference's module names, state_dict keys and ``get_config()``, the input and the output.  Weights are not stored: they are
regenerated from the seed.
"""
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("GALRNET_REF_SRC", "/root/reference/src")
sys.path.insert(0, REF_SRC)
sys.path.insert(0, os.path.dirname(HERE))
warnings.simplefilter("ignore")
from models.galrnet import GALRNet  # noqa: E402  (reference)

import galrnet_ref as R  # noqa: E402

RECIPE = dict(n_basis=64, kernel_size=16, stride=8, enc_nonlinear=None, sep_hidden_channels=128, sep_chunk_size=100, sep_hop_size=50,
              sep_down_chunk_size=32, sep_num_blocks=6, sep_num_heads=8, sep_dropout=0.1, mask_nonlinear="relu", eps=1e-12)
CASES = {
    "tiny": dict(n_basis=32, kernel_size=4, stride=2, enc_nonlinear="relu", sep_hidden_channels=32, sep_chunk_size=16, sep_hop_size=8,
                 sep_down_chunk_size=4, sep_num_blocks=2, sep_num_heads=4, sep_dropout=0.1, mask_nonlinear="sigmoid", eps=1e-12,
                 n_sources=2, batch=2, T=301, seed=21),
    # 4000 samples: 499 frames, S = 9 chunks
    "recipe_2spk": dict(RECIPE, n_sources=2, batch=1, T=4000, seed=22),
    "recipe_3spk": dict(RECIPE, n_sources=3, batch=2, T=3000, seed=23),
    # 808 samples: 100 frames, one chunk (S = 1)
    "single_chunk": dict(RECIPE, n_sources=2, batch=1, T=808, seed=24),
}


def build(cfg):
    return GALRNet(cfg["n_basis"], cfg["kernel_size"], stride=cfg["stride"], enc_basis="trainable", dec_basis="trainable",
                   enc_nonlinear=cfg["enc_nonlinear"], sep_hidden_channels=cfg["sep_hidden_channels"], sep_chunk_size=cfg["sep_chunk_size"],
                   sep_hop_size=cfg["sep_hop_size"], sep_down_chunk_size=cfg["sep_down_chunk_size"], sep_num_blocks=cfg["sep_num_blocks"],
                   sep_num_heads=cfg["sep_num_heads"], sep_norm=True, sep_dropout=cfg["sep_dropout"], mask_nonlinear=cfg["mask_nonlinear"],
                   low_dimension=True, causal=False, n_sources=cfg["n_sources"], eps=cfg["eps"])


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
                     "ref_config": model.get_config(), "num_parameters": model.num_parameters, "x": x, "out": y}
        print(name, tuple(y.shape), float(y.abs().max()), model.num_parameters, len(keys_shapes))
    torch.save(out, os.path.join(HERE, "galrnet.pt"))


if __name__ == "__main__":
    main()
