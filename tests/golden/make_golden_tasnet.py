#!/usr/bin/env python
"""Mint LSTM-TasNet golden vectors from the UNMODIFIED reference (run where the reference's src/ is available).

    python tests/golden/make_golden_tasnet.py          # writes tests/golden/tasnet.pt

The reference's TasNet is built as-is, loaded with seeded weights from tests/lstm_tasnet_ref.py (``synth_state_dict``) through
``load_state_dict(strict=True)`` and run in fp32 on the CPU in eval mode.  Stored per case: the config, the seed, the reference's
module names and state_dict keys, the input and the output, and the reference's own ``get_config()`` (the checkpoint header its
trainer writes).  Weights are not stored: they are regenerated from the seed.
"""
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("TASNET_REF_SRC", "/root/reference/src")
sys.path.insert(0, REF_SRC)
sys.path.insert(0, os.path.dirname(HERE))
warnings.simplefilter("ignore")
from models.tasnet import TasNet  # noqa: E402  (reference)

import lstm_tasnet_ref as R  # noqa: E402

RECIPE = dict(n_basis=500, kernel_size=40, stride=20, enc_basis="trainableGated", enc_nonlinear=None, sep_num_blocks=2, sep_num_layers=2,
              sep_hidden_channels=500, causal=False, mask_nonlinear="sigmoid", eps=1e-12)
CASES = {
    "tiny_gated": dict(n_basis=32, kernel_size=16, stride=8, enc_basis="trainableGated", enc_nonlinear=None, sep_num_blocks=2,
                       sep_num_layers=2, sep_hidden_channels=24, causal=False, mask_nonlinear="sigmoid", eps=1e-12, n_sources=2, batch=2,
                       T=1003, seed=31),
    "tiny_plain_softmax": dict(n_basis=24, kernel_size=8, stride=4, enc_basis="trainable", enc_nonlinear="relu", sep_num_blocks=2,
                               sep_num_layers=1, sep_hidden_channels=16, causal=False, mask_nonlinear="softmax", eps=1e-12, n_sources=3,
                               batch=2, T=517, seed=32),
    "tiny_causal": dict(n_basis=32, kernel_size=16, stride=8, enc_basis="trainableGated", enc_nonlinear=None, sep_num_blocks=2,
                        sep_num_layers=2, sep_hidden_channels=20, causal=True, mask_nonlinear="sigmoid", eps=1e-12, n_sources=2, batch=2,
                        T=800, seed=33),
    "recipe_2spk": dict(RECIPE, n_sources=2, batch=1, T=16000, seed=34),
    "recipe_3spk": dict(RECIPE, n_sources=3, batch=2, T=6001, seed=35),
}


def build(cfg):
    return TasNet(cfg["n_basis"], kernel_size=cfg["kernel_size"], stride=cfg["stride"], enc_basis=cfg["enc_basis"], dec_basis="trainable",
                  enc_nonlinear=cfg["enc_nonlinear"], sep_num_blocks=cfg["sep_num_blocks"], sep_num_layers=cfg["sep_num_layers"],
                  sep_hidden_channels=cfg["sep_hidden_channels"], mask_nonlinear=cfg["mask_nonlinear"], causal=cfg["causal"],
                  rnn_type="lstm", n_sources=cfg["n_sources"], eps=cfg["eps"])


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
        print(name, tuple(y.shape), float(y.abs().max()))
    torch.save(out, os.path.join(HERE, "tasnet.pt"))


if __name__ == "__main__":
    main()
