"""GALRNet without a GPU: the fp64 restatement against the reference's goldens, the module tree and state_dict keys, a checkpoint
in the recipe trainer's format, every envelope refusal (before any CUDA check), and the planted defects the GPU bound must
reject."""
import os

import pytest
import torch

import galrnet_ref as R
from ctn_b200.models import galr as G
from ctn_b200.models.dprnn import IntraChunkRNN
from ctn_b200.models.galrnet import GALRNet

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "galrnet.pt"), weights_only=False)


def make(cfg, **over):
    kw = dict(stride=cfg["stride"], enc_basis="trainable", dec_basis="trainable", enc_nonlinear=cfg["enc_nonlinear"],
              sep_hidden_channels=cfg["sep_hidden_channels"], sep_chunk_size=cfg["sep_chunk_size"], sep_hop_size=cfg["sep_hop_size"],
              sep_down_chunk_size=cfg["sep_down_chunk_size"], sep_num_blocks=cfg["sep_num_blocks"], sep_num_heads=cfg["sep_num_heads"],
              sep_norm=True, sep_dropout=cfg["sep_dropout"], mask_nonlinear=cfg["mask_nonlinear"], low_dimension=True, causal=False,
              n_sources=cfg["n_sources"], eps=cfg["eps"])
    kw.update(over)
    return GALRNet(cfg["n_basis"], cfg["kernel_size"], **kw)


@pytest.mark.parametrize("case", sorted(GOLD))
def test_fp64_restatement_matches_reference(case):
    g = GOLD[case]
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    out = R.galrnet_fwd(g["x"], sd, g["cfg"])
    ref = g["out"].double()
    assert out.shape == ref.shape
    # the goldens come from the reference in fp32
    assert float((out - ref).abs().max()) < 2e-5 * float(ref.abs().max())


def test_encoding_is_the_references_fp32_table():
    """the divisors the kernel divides by are the reference's fp32 values; sin / cos of their quotients give its table"""
    blk = G.LowDimensionGloballyAttentiveBlock(64, chunk_size=100, down_chunk_size=32, num_heads=8)
    F, n = 64, 79 * 32
    div = blk.pe_divisors(F)
    assert div.dtype == torch.float32 and div.shape == (F // 2,)
    assert torch.equal(div, 10000 ** (torch.arange(F // 2) / F))
    assert torch.equal(blk.positional_encoding(n, F).double(), R.pe_table(n, F))


@pytest.mark.parametrize("case", sorted(GOLD))
def test_module_tree_and_keys_equal_reference(case):
    g = GOLD[case]
    m = make(g["cfg"])
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in g["keys_shapes"]]
    assert m.num_parameters == g["num_parameters"]
    # the separator's tree; the filter banks are the package's shared Encoder / Decoder, whose parameters match above
    sep = lambda mods: [(n, t) for n, t in mods if n.startswith("separator")]  # noqa: E731
    assert sep([(n, type(x).__name__) for n, x in m.named_modules()]) == sep(g["modules"])
    assert all(type(b.intra_chunk_block) is IntraChunkRNN for b in m.separator.galr.net)
    m.load_state_dict(R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"]), strict=True)


def test_recipe_size():
    g = GOLD["recipe_2spk"]
    assert g["num_parameters"] == 1450777 and len(g["keys_shapes"]) == 155
    assert not any("_pe_div" in k for k, _ in make(g["cfg"]).named_buffers())


def test_trainer_checkpoint_round_trip(tmp_path):
    """the recipe's trainer saves get_config() plus 'state_dict' (adhoc_driver.py:208-214); GALRNet(**config) loads it strictly"""
    g = GOLD["recipe_3spk"]
    sd = R.synth_state_dict(g["keys_shapes"], 3)
    ckpt = dict(g["ref_config"])
    ckpt["state_dict"] = sd
    path = str(tmp_path / "best.pth")
    torch.save(ckpt, path)
    config = torch.load(path, map_location="cpu", weights_only=False)
    state = config.pop("state_dict")
    m = GALRNet(**config)
    m.load_state_dict(state, strict=True)
    assert m.get_config() == g["ref_config"]
    for k, v in sd.items():
        assert torch.equal(m.state_dict()[k], v)
    assert not hasattr(GALRNet, "build_model") and not hasattr(GALRNet, "build_from_pretrained")


@pytest.mark.parametrize("over,exc", [
    (dict(causal=True), NotImplementedError),
    (dict(low_dimension=False), NotImplementedError),
    (dict(sep_norm=False), NotImplementedError),
    (dict(mask_nonlinear="softmax"), NotImplementedError),
    (dict(mask_nonlinear="tanh"), ValueError),
    (dict(enc_basis="Fourier", dec_basis="Fourier", window_fn="hann", enc_onesided=True, enc_return_complex=True), NotImplementedError),
    (dict(in_channels=2), NotImplementedError),
    (dict(sep_num_heads=8), NotImplementedError),               # head dimension 32 / 8 = 4
    (dict(sep_down_chunk_size=17), NotImplementedError),        # Q > K
    (dict(sep_hidden_channels=48), NotImplementedError),        # outside the LSTM kernel's sizes
    (dict(sep_down_chunk_size=None), ValueError),
])
def test_envelope_refusals(over, exc):
    with pytest.raises(exc):
        make(GOLD["tiny"]["cfg"], **over)


def test_features_outside_kernel_envelope_refused():
    with pytest.raises(NotImplementedError):
        G.LowDimensionGloballyAttentiveBlock(48, chunk_size=16, down_chunk_size=4, num_heads=6)
    with pytest.raises(NotImplementedError):
        G.GloballyAttentiveBlock(32, num_heads=4)


def test_forward_and_launch_limit_refusals_before_cuda():
    g = GOLD["tiny"]
    m = make(g["cfg"]).eval()
    x = g["x"]  # CPU tensors: every refusal must fire before the CUDA check
    with pytest.raises(NotImplementedError, match="forward-only"):
        m(x)
    with torch.no_grad():
        with pytest.raises(ValueError):
            m(x[:, 0])
        with pytest.raises(ValueError, match="too short"):
            m(x[..., :10])
    m.train()
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="dropout"):
            m(x)
    sep = m.separator
    blk = sep.galr.net[0]
    z = torch.randn(2, 32, 3, 16)
    with pytest.raises(NotImplementedError, match="forward-only"):
        blk(z)
    with pytest.raises(NotImplementedError, match="forward-only"):
        blk.inter_chunk_block(z)
    with pytest.raises(NotImplementedError, match="forward-only"):
        sep.galr(z)
    with torch.no_grad():
        with pytest.raises(NotImplementedError, match="dropout"):
            blk.inter_chunk_block(z)
        with pytest.raises(NotImplementedError):
            sep(torch.randn(2, 32, 50))
        with pytest.raises(NotImplementedError):
            blk.inter_chunk_block.norm2d_in(z)
    m.eval()
    with torch.no_grad(), pytest.raises(NotImplementedError, match="launch limits"):
        blk.inter_chunk_block.check_shape((65536, 3, 16, 32))  # batch_size > 65535: the grids of the down- and up-map
    with torch.no_grad(), pytest.raises(NotImplementedError, match="launch limits"):
        blk.inter_chunk_block.check_shape((2, 65536, 16, 32))    # S > 65535
    blk.inter_chunk_block.check_shape((16385, 3, 16, 32))  # batch_size * down_chunk_size > 65535: the attention takes any count
    with torch.no_grad(), pytest.raises(ValueError):
        blk.inter_chunk_block(torch.randn(2, 32, 3, 15))       # not the chunk size the block was built for


@pytest.mark.parametrize("defect", R.DEFECTS)
def test_bound_rejects_planted_defects(defect):
    g = GOLD["tiny"]
    cfg = dict(g["cfg"])
    sd = R.synth_state_dict(g["keys_shapes"], cfg["seed"])
    # 1400 samples: 699 frames, S = 87 chunks
    x = torch.randn(1, 1, 1400, generator=torch.Generator().manual_seed(5))
    ref = R.galrnet_fwd(x, sd, cfg)
    bad = R.galrnet_fwd(x, sd, cfg, defect=defect)
    assert float((bad - ref).abs().max()) > 10 * R.bound(ref), defect
