"""DPTNet without a GPU: the fp64 restatement against the reference's goldens, the module tree and state_dict keys, the
config round trip, every envelope refusal (before any CUDA check), and the planted defects the GPU bound must reject."""
import os
import sys
import types

import pytest
import torch

import dptnet_ref as R
from ctn_b200.models.dptnet import DPTNet
from ctn_b200.models.gtu import GTU1d

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dptnet.pt"), weights_only=False)


def make(cfg, **over):
    kw = dict(enc_basis="trainable", dec_basis="trainable", enc_nonlinear=cfg["enc_nonlinear"], stride=cfg["stride"],
              sep_bottleneck_channels=cfg["sep_bottleneck_channels"], sep_hidden_channels=cfg["sep_hidden_channels"],
              sep_chunk_size=cfg["sep_chunk_size"], sep_hop_size=cfg["sep_hop_size"], sep_num_blocks=cfg["sep_num_blocks"],
              sep_num_heads=cfg["sep_num_heads"], mask_nonlinear=cfg["mask_nonlinear"], causal=False, n_sources=cfg["n_sources"],
              eps=cfg["eps"])
    kw.update(over)
    return DPTNet(cfg["n_basis"], cfg["kernel_size"], **kw)


@pytest.mark.parametrize("case", sorted(GOLD))
def test_fp64_restatement_matches_reference(case):
    g = GOLD[case]
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    out = R.dptnet_fwd(g["x"], sd, g["cfg"])
    ref = g["out"].double()
    assert out.shape == ref.shape
    # the goldens come from the reference in fp32
    assert float((out - ref).abs().max()) < 2e-5 * float(ref.abs().max())


@pytest.mark.parametrize("case", sorted(GOLD))
def test_module_tree_and_keys_equal_reference(case):
    g = GOLD[case]
    m = make(g["cfg"])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in g["keys_shapes"]]
    # the separator's tree; the filter banks are the package's shared Encoder / Decoder, whose parameters match above
    sep = lambda mods: [(n, t) for n, t in mods if n.startswith("separator")]  # noqa: E731
    assert sep([(n, type(x).__name__) for n, x in m.named_modules()]) == sep(g["modules"])
    m.load_state_dict(R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"]), strict=True)


def test_build_model_round_trip(tmp_path):
    g = GOLD["tiny"]
    m = make(g["cfg"], sep_dropout=0.1)
    m.load_state_dict(R.synth_state_dict(g["keys_shapes"], 3))
    path = str(tmp_path / "m.pth")
    cfg = m.get_config()
    cfg["state_dict"] = m.state_dict()
    torch.save(cfg, path)
    m2 = DPTNet.build_model(path, load_state_dict=True)
    assert m2.get_config() == m.get_config()
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k])
    with pytest.raises(FileNotFoundError):
        DPTNet.build_from_pretrained(root=str(tmp_path), task="wsj0-mix", n_sources=2)
    with pytest.raises(KeyError):
        DPTNet.build_from_pretrained(root=str(tmp_path), task="musdb18")


def test_build_from_pretrained_never_downloads(tmp_path, monkeypatch):
    """a missing checkpoint names its path even where the reference's downloader is importable, and the downloader is not called"""
    def download(*args, **kwargs):
        pytest.fail("build_from_pretrained called a downloader")
    utils = types.ModuleType("utils")
    utils.utils = types.ModuleType("utils.utils")
    utils.utils.download_pretrained_model_from_google_drive = download
    monkeypatch.setitem(sys.modules, "utils", utils)
    monkeypatch.setitem(sys.modules, "utils.utils", utils.utils)
    with pytest.raises(FileNotFoundError, match=os.path.join("DPTNet", "wsj0-mix", "sr8000", "2speakers", "model", "best.pth")):
        DPTNet.build_from_pretrained(root=str(tmp_path), task="wsj0-mix", n_sources=2)


@pytest.mark.parametrize("over,exc", [
    (dict(causal=True), NotImplementedError),
    (dict(mask_nonlinear="softmax"), NotImplementedError),
    (dict(mask_nonlinear="tanh"), ValueError),
    (dict(sep_nonlinear="gelu"), NotImplementedError),
    (dict(sep_norm=False), NotImplementedError),
    (dict(sep_hidden_channels=48), NotImplementedError),       # outside the LSTM kernel's sizes
    (dict(sep_num_heads=1), NotImplementedError),              # head dimension 32 * 4 = 128 with F = 128 below
    (dict(enc_basis="Fourier", dec_basis="Fourier", window_fn="hann", enc_onesided=True, enc_return_complex=True), NotImplementedError),
    (dict(in_channels=2), NotImplementedError),
])
def test_envelope_refusals(over, exc):
    cfg = dict(GOLD["tiny"]["cfg"])
    if over.get("sep_num_heads") == 1:
        cfg.update(n_basis=128, sep_bottleneck_channels=128)
    with pytest.raises(exc):
        make(cfg, **over)


def test_head_dimension_not_multiple_of_8_refused():
    cfg = dict(GOLD["tiny"]["cfg"])
    cfg.update(sep_num_heads=8)  # 32 / 8 = 4
    with pytest.raises(NotImplementedError):
        make(cfg)


def test_forward_refusals_before_cuda():
    g = GOLD["tiny"]
    m = make(g["cfg"])
    x = g["x"]  # a CPU tensor: the refusals must fire before the CUDA check
    with pytest.raises(NotImplementedError, match="forward-only"):
        m(x)
    frozen = make(g["cfg"]).requires_grad_(False)             # no parameter requires grad, the input does
    with pytest.raises(NotImplementedError, match="forward-only"):
        frozen(x.clone().requires_grad_())
    with torch.no_grad():
        with pytest.raises(ValueError):
            m(x[:, 0])
    md = make(g["cfg"], sep_dropout=0.1)
    md.train()
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="dropout"):
            md(x)
    with pytest.raises(NotImplementedError):
        GTU1d(4, 4, kernel_size=3)


@pytest.mark.parametrize("defect", R.DEFECTS)
def test_bound_rejects_planted_defects(defect):
    g = GOLD["tiny"]
    cfg = dict(g["cfg"])
    sd = R.synth_state_dict(g["keys_shapes"], cfg["seed"])
    # 1400 samples: 699 frames, S = 87 chunks, so the inter-chunk attention has a second (partial) key tile
    x = torch.randn(1, 1, 1400, generator=torch.Generator().manual_seed(5))
    ref = R.dptnet_fwd(x, sd, cfg)
    bad = R.dptnet_fwd(x, sd, cfg, defect=defect)
    assert float((bad - ref).abs().max()) > 10 * R.bound(ref), defect
