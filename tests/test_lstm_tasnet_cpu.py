"""LSTM-TasNet without a GPU: the fp64 restatement against the reference's goldens, the module tree and state_dict keys, the config
round trip, every refusal that comes before any CUDA work, the other models' refusal of the gated encoder, and the planted defects
the GPU bound must reject."""
import os

import pytest
import torch

import lstm_tasnet_ref as R
from ctn_b200.models.tasnet import TasNet
from ctn_b200.models.lstm_tasnet import LSTMTasNet
from ctn_b200.models.conv_tasnet import ConvTasNet
from ctn_b200.models.dprnn_tasnet import DPRNNTasNet
from ctn_b200.models.dptnet import DPTNet
from ctn_b200.models.sepformer import SepFormer
from ctn_b200.models.filterbank import GatedEncoder

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tasnet.pt"), weights_only=False)
ARGS = ("kernel_size", "stride", "enc_basis", "enc_nonlinear", "sep_num_blocks", "sep_num_layers", "sep_hidden_channels", "causal",
        "mask_nonlinear", "n_sources", "eps")


def make(cfg, **over):
    kw = dict(dec_basis="trainable", rnn_type="lstm", **{k: cfg[k] for k in ARGS})
    kw.update(over)
    return TasNet(cfg["n_basis"], **kw)


@pytest.mark.parametrize("case", sorted(GOLD))
def test_fp64_restatement_matches_reference(case):
    g = GOLD[case]
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    out = R.tasnet_fwd(g["x"], sd, g["cfg"])
    ref = g["out"].double()
    assert out.shape == ref.shape
    # the goldens come from the reference in fp32
    assert float((out - ref).abs().max()) < 2e-5 * float(ref.abs().max())


@pytest.mark.parametrize("case", sorted(GOLD))
def test_module_tree_and_keys_equal_reference(case):
    g = GOLD[case]
    m = make(g["cfg"])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in g["keys_shapes"]]
    # the shared plain Encoder applies its ReLU inside the kernel and holds no nonlinear1d module (no parameters, no keys)
    ref_modules = [(n, t) for n, t in g["modules"] if n != "encoder.nonlinear1d"]
    assert [(n, type(x).__name__) for n, x in m.named_modules()] == ref_modules
    assert m.num_parameters == g["num_parameters"]
    assert m.get_config() == g["ref_config"]
    m.load_state_dict(R.synth_state_dict(g["keys_shapes"], 1), strict=True)


def test_recipe_keys():
    keys = [k for k, _ in GOLD["recipe_2spk"]["keys_shapes"]]
    assert keys[:2] == ["encoder.conv1d_U.weight", "encoder.conv1d_V.weight"]
    assert "separator.gamma" in keys and "separator.beta" in keys and "decoder.conv_transpose1d.weight" in keys
    for blk in range(2):
        for layer in range(2):
            for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                for sfx in ("", "_reverse"):
                    assert "separator.rnn.{}.{}_l{}{}".format(blk, n, layer, sfx) in keys
    assert dict(GOLD["recipe_2spk"]["keys_shapes"])["separator.fc.weight"] == (1000, 1000)
    assert dict(GOLD["recipe_3spk"]["keys_shapes"])["separator.fc.weight"] == (1500, 1000)
    assert LSTMTasNet is TasNet
    from models.lstm_tasnet import LSTMTasNet as shim_alias  # the drop-in shim
    from models.tasnet import TasNet as shim_cls
    assert shim_alias is TasNet and shim_cls is TasNet


def test_build_model_round_trip(tmp_path):
    g = GOLD["tiny_gated"]
    m = make(g["cfg"])
    m.load_state_dict(R.synth_state_dict(g["keys_shapes"], 3))
    path = str(tmp_path / "m.pth")
    cfg = m.get_config()
    cfg["state_dict"] = m.state_dict()
    torch.save(cfg, path)
    m2 = TasNet.build_model(path, load_state_dict=True)
    assert m2.get_config() == m.get_config()
    for k, v in m.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k])
    # the legacy keys of older checkpoints
    legacy = dict(cfg)
    legacy["n_bases"], legacy["enc_bases"], legacy["dec_bases"] = legacy.pop("n_basis"), legacy.pop("enc_basis"), legacy.pop("dec_basis")
    del legacy["rnn_type"], legacy["in_channels"]
    torch.save(legacy, path)
    m3 = TasNet.build_model(path, load_state_dict=True)
    assert m3.get_config() == m.get_config()
    with pytest.raises(FileNotFoundError, match=os.path.join("TasNet", "wsj0-mix", "sr8000", "2speakers", "model", "best.pth")):
        TasNet.build_from_pretrained(root=str(tmp_path), task="wsj0-mix", n_sources=2)
    with pytest.raises(KeyError):
        TasNet.build_from_pretrained(root=str(tmp_path), task="musdb18")


def test_plain_encoder_config_round_trip(tmp_path):
    g = GOLD["tiny_plain_softmax"]
    m = make(g["cfg"])
    path = str(tmp_path / "p.pth")
    cfg = m.get_config()
    cfg["state_dict"] = m.state_dict()
    torch.save(cfg, path)
    # the reference's get_config() has no enc_nonlinear: a rebuilt plain encoder has none either, as in the reference
    assert TasNet.build_model(path, load_state_dict=True).encoder.nonlinear is False


def test_refusals_before_cuda():
    g = GOLD["tiny_gated"]
    x = torch.randn(1, 1, 400)
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="rnn_type"):
            make(g["cfg"], rnn_type="gru")(x)
        with pytest.raises(NotImplementedError, match="4-D"):
            make(g["cfg"])(x.view(1, 1, 1, 400))
        with pytest.raises(NotImplementedError, match="multichannel"):
            make(g["cfg"], in_channels=2)(x)
        with pytest.raises(ValueError, match="too short"):
            make(g["cfg"])(torch.randn(1, 1, 8))  # padded to 8 < kernel_size 16
        with pytest.raises(ValueError):
            make(g["cfg"])(torch.randn(1, 400))
    with pytest.raises(NotImplementedError, match="forward-only"):
        make(g["cfg"])(x)
    with pytest.raises(NotImplementedError, match="not built"):
        make(g["cfg"]).separator(torch.randn(1, 32, 10))
    with pytest.raises(AssertionError):
        make(g["cfg"], enc_basis="Fourier")


def test_other_models_still_refuse_gated_encoder():
    with pytest.raises(NotImplementedError, match="trainableGated"):
        ConvTasNet(64, 16, enc_basis="trainableGated", dec_basis="trainable", sep_hidden_channels=64, sep_bottleneck_channels=32,
                   sep_skip_channels=32, sep_num_blocks=1, sep_num_layers=2, causal=False)
    with pytest.raises(NotImplementedError, match="trainableGated"):
        DPRNNTasNet(64, 16, enc_basis="trainableGated", dec_basis="trainable", sep_hidden_channels=64, sep_bottleneck_channels=64,
                    sep_chunk_size=10, sep_hop_size=5, sep_num_blocks=1, causal=False)
    with pytest.raises(NotImplementedError, match="trainableGated"):
        DPTNet(64, 16, enc_basis="trainableGated", dec_basis="trainable", sep_bottleneck_channels=64, sep_hidden_channels=64,
               sep_chunk_size=10, sep_hop_size=5, sep_num_blocks=1, sep_num_heads=4, causal=False)
    with pytest.raises(NotImplementedError, match="trainableGated"):
        SepFormer(64, 16, enc_basis="trainableGated", dec_basis="trainable", sep_bottleneck_channels=64, sep_chunk_size=10,
                  sep_hop_size=5, sep_num_blocks=1, causal=False)


def test_gated_encoder_module():
    e = GatedEncoder(1, 8, kernel_size=4, stride=2)
    assert [n for n, _ in e.named_parameters()] == ["conv1d_U.weight", "conv1d_V.weight"]
    assert e.eps == 1e-12
    with pytest.raises(ValueError):
        e(torch.randn(2, 3, 10))


@pytest.mark.parametrize("defect", R.DEFECTS)
def test_bound_rejects_planted_defect(defect):
    case = "tiny_plain_softmax" if defect in ("softmax_channels",) else "tiny_gated"
    g = GOLD[case]
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    ref = R.tasnet_fwd(g["x"], sd, g["cfg"])
    bad = R.tasnet_fwd(g["x"], sd, g["cfg"], defect=defect)
    assert float((bad - ref).abs().max()) > 10 * R.bound(ref), defect
