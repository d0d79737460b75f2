"""SepFormer without a GPU: the fp64 restatement against the reference's goldens, the module tree, state_dict keys and buffers,
the config round trip, every envelope refusal (before any CUDA check), and the planted defects the GPU bound must reject."""
import os

import pytest
import torch

import sepformer_ref as R
from ctn_b200.models.sepformer import SepFormer
from ctn_b200.models.transformer import PositionalEncoding

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sepformer.pt"), weights_only=False)
ARGS = ("stride", "enc_nonlinear", "sep_bottleneck_channels", "sep_chunk_size", "sep_hop_size", "sep_num_blocks", "sep_num_layers_intra",
        "sep_num_layers_inter", "sep_num_heads_intra", "sep_num_heads_inter", "sep_d_ff_intra", "sep_d_ff_inter", "mask_nonlinear",
        "n_sources", "eps")


def make(cfg, **over):
    kw = dict(enc_basis="trainable", dec_basis="trainable", causal=False, **{k: cfg[k] for k in ARGS})
    kw.update(over)
    return SepFormer(cfg["n_basis"], cfg["kernel_size"], **kw)


@pytest.mark.parametrize("case", sorted(GOLD))
def test_fp64_restatement_matches_reference(case):
    g = GOLD[case]
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    out = R.sepformer_fwd(g["x"], sd, g["cfg"])
    ref = g["out"].double()
    assert out.shape == ref.shape
    # the goldens come from the reference in fp32
    assert float((out - ref).abs().max()) < 2e-5 * float(ref.abs().max())


@pytest.mark.parametrize("case", sorted(GOLD))
def test_module_tree_keys_and_buffers_equal_reference(case):
    g = GOLD[case]
    m = make(g["cfg"])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in g["keys_shapes"]]
    sep = lambda mods: [(n, t) for n, t in mods if n.startswith("separator")]  # noqa: E731
    assert sep([(n, type(x).__name__) for n, x in m.named_modules()]) == sep(g["modules"])
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    pe_keys = [k for k in sd if k.endswith(R.PE_KEY)]
    assert len(pe_keys) == 2 * g["cfg"]["sep_num_blocks"]
    for k in pe_keys:  # the module builds the reference's buffer bit for bit
        assert torch.equal(m.state_dict()[k], sd[k]), k
    m.load_state_dict(sd, strict=True)


def test_recipe_key_count():
    assert len(GOLD["recipe_2spk"]["keys_shapes"]) == 411
    keys = [k for k, _ in GOLD["recipe_2spk"]["keys_shapes"]]
    assert sum(k.endswith("transformer.norm.norm1d.norm.weight") for k in keys) == 4
    assert all(tuple(s) == (5000, 1, 256) for k, s in GOLD["recipe_2spk"]["keys_shapes"] if k.endswith(R.PE_KEY))


def test_positional_encoding_is_interleaved():
    pe = PositionalEncoding(8).positional_encoding
    assert pe.shape == (5000, 1, 8)
    t = torch.arange(5000, dtype=torch.float64)
    for i in range(4):
        w = 10000.0 ** (2 * i / 8)
        assert torch.allclose(pe[:, 0, 2 * i].double(), torch.sin(t / w), atol=1e-3)
        assert torch.allclose(pe[:, 0, 2 * i + 1].double(), torch.cos(t / w), atol=1e-3)


def test_build_model_round_trip(tmp_path):
    g = GOLD["tiny"]
    m = make(g["cfg"], sep_dropout=0.1)
    m.load_state_dict(R.synth_state_dict(g["keys_shapes"], 3))
    path = str(tmp_path / "m.pth")
    cfg = m.get_config()
    cfg["state_dict"] = m.state_dict()
    torch.save(cfg, path)
    m2 = SepFormer.build_model(path, load_state_dict=True)
    assert m2.get_config() == m.get_config()
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k])
    with pytest.raises(FileNotFoundError, match=os.path.join("SepFormer", "wsj0-mix", "sr8000", "2speakers", "model", "best.pth")):
        SepFormer.build_from_pretrained(root=str(tmp_path), task="wsj0-mix", n_sources=2)
    with pytest.raises(KeyError):
        SepFormer.build_from_pretrained(root=str(tmp_path), task="musdb18")


@pytest.mark.parametrize("over,exc", [
    (dict(causal=True), NotImplementedError),
    (dict(mask_nonlinear="softmax"), NotImplementedError),
    (dict(mask_nonlinear="tanh"), ValueError),
    (dict(sep_nonlinear="gelu"), NotImplementedError),
    (dict(sep_norm=False), NotImplementedError),
    (dict(sep_num_heads_intra=8), NotImplementedError),        # 32 / 8 = 4: not a supported head dimension
    (dict(sep_num_heads_inter=1), NotImplementedError),        # 32 / 1 = 32 is fine, checked below with F = 256
    (dict(enc_basis="Fourier", dec_basis="Fourier", window_fn="hann", enc_onesided=True, enc_return_complex=True), NotImplementedError),
    (dict(in_channels=2), NotImplementedError),
])
def test_envelope_refusals(over, exc):
    cfg = dict(GOLD["tiny"]["cfg"])
    if over.get("sep_num_heads_inter") == 1:
        cfg.update(n_basis=256, sep_bottleneck_channels=256)  # head dimension 256
    with pytest.raises(exc):
        make(cfg, **over)


def test_causal_refusal_names_the_switch():
    with pytest.raises(NotImplementedError, match="causal=False"):
        SepFormer(32, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear="relu", sep_num_heads_intra=4,
                  sep_num_heads_inter=4)


def test_intra_and_inter_heads_checked_separately():
    cfg = dict(GOLD["tiny"]["cfg"])
    make(cfg, sep_num_heads_intra=2, sep_num_heads_inter=4)   # 16 and 8
    with pytest.raises(NotImplementedError):
        make(cfg, sep_num_heads_intra=2, sep_num_heads_inter=16)  # inter head dimension 2


def test_forward_refusals_before_cuda():
    g = GOLD["tiny"]
    m = make(g["cfg"]).eval()
    x = g["x"]  # a CPU tensor: the refusals must fire before the CUDA check
    with pytest.raises(NotImplementedError, match="forward-only"):
        m(x)
    with torch.no_grad():
        with pytest.raises(ValueError):
            m(x[:, 0])
        with pytest.raises(ValueError, match="too short"):
            m(x[:, :, :40])                                   # 4 frames + 4 of padding < one chunk of 16
        with pytest.raises(ValueError, match="positional encoding"):
            m(torch.zeros(1, 1, 8 * 40016 + 8))               # 40016 frames: 5001 chunks
        with pytest.raises(ValueError, match="positional encoding"):
            make(g["cfg"], sep_chunk_size=5001, sep_hop_size=2500).eval()(torch.zeros(1, 1, 8 * 5001 + 8))
    md = make(g["cfg"], sep_dropout=0.1)
    md.train()
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="dropout"):
            md(x)


@pytest.mark.parametrize("defect", R.DEFECTS)
def test_bound_rejects_planted_defects(defect):
    g = GOLD["tiny"]
    cfg = dict(g["cfg"])
    sd = R.synth_state_dict(g["keys_shapes"], cfg["seed"])
    x = torch.randn(1, 1, 2000, generator=torch.Generator().manual_seed(5))
    ref = R.sepformer_fwd(x, sd, cfg)
    bad = R.sepformer_fwd(x, sd, cfg, defect=defect)
    assert float((bad - ref).abs().max()) > 10 * R.bound(ref), defect
