#!/usr/bin/env python
"""Mint the causal plain-encoder LSTM-TasNet golden vectors (the model that streams) from the UNMODIFIED reference (run where the
reference's src/ is available).

    python tests/golden/make_golden_tasnet_causal_plain.py          # writes tests/golden/tasnet_causal_plain.pt

As make_golden_tasnet.py: the reference's TasNet is built as-is, loaded with seeded weights from tests/lstm_tasnet_ref.py
(``synth_state_dict``) through ``load_state_dict(strict=True)`` and run in fp32 on the CPU in eval mode.  T is a multiple of the
stride, where the reference adds no padding.  Weights are not stored: they are regenerated from the seed.
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

CASES = {
    "causal_plain_sigmoid": dict(n_basis=32, kernel_size=16, stride=8, enc_basis="trainable", enc_nonlinear=None, sep_num_blocks=2,
                                 sep_num_layers=2, sep_hidden_channels=24, causal=True, mask_nonlinear="sigmoid", eps=1e-12, n_sources=2,
                                 batch=2, T=800, seed=41),
    "causal_plain_softmax": dict(n_basis=24, kernel_size=8, stride=4, enc_basis="trainable", enc_nonlinear="relu", sep_num_blocks=3,
                                 sep_num_layers=1, sep_hidden_channels=16, causal=True, mask_nonlinear="softmax", eps=1e-12, n_sources=3,
                                 batch=2, T=520, seed=42),
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
        out[name] = {"cfg": cfg, "keys_shapes": keys_shapes, "ref_config": model.get_config(), "x": x, "out": y}
        print(name, tuple(y.shape), float(y.abs().max()))
    torch.save(out, os.path.join(HERE, "tasnet_causal_plain.pt"))


if __name__ == "__main__":
    main()
