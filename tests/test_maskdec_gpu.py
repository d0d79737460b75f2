"""The fused mask + decoder launch (k_maskdec: ctn_pw(..., PRO_PRELU, EPI_MASKDEC, f16x3)) across sources, basis sizes, operand
widths, tile edges, crops and batch sizes (``-m gpu``).

Each row goes through the verification hook with the helpers of test_pw_contraction_gpu.py: the estimates pass the fp64 gate of
pw_criterion.epi_maskdec, and a second call gives the same bits.  K = 129, one channel past the resident operand's limit, must be
refused by the launch.  At model level, a forward with skip <= 128 (fused) is compared with extract_latent (always the unfused
mask + decoder) and with the CPU oracle; with skip = 160 both calls take the unfused path (the fallback), which is held to the
oracle.
"""
import pytest
import torch

import convtasnet_oracle as O
import test_pw_contraction_gpu as PW
from ctn_b200 import _native as N

pytestmark = pytest.mark.gpu


def _md(S, Nb, K, frames, crop, B, reaches, **kw):
    return PW._row("prelu", "maskdec", S * Nb, K, frames, reaches, B=B, Nb=Nb, crop=crop, modes=["f16x3"], **kw)


ROWS = {
    "s1_nb128_k33_f1": _md(1, 128, 33, 1, 0, 1, "one frame, one n-tile, a 1-channel last slab"),
    "s2_nb128_k96_f127_b3": _md(2, 128, 96, 127, 4, 3, "two sources of one n-tile each, frames one short of a tile"),
    "s3_nb256_k128_f128": _md(3, 256, 128, 128, 0, 1, "S = 3: six n-tiles, one full tile, K at the resident limit"),
    "s4_nb512_k128_f129_b3": _md(4, 512, 128, 129, 4, 3, "S = 4 x 4 n-tiles = M 2048: the ring across sources, a seam"),
    "s2_nb512_k128_f3999": _md(2, 512, 128, 3999, 4, 1, "the cfg2 shape of one sample: 32 tiles"),
    "s4_nb256_k33_f1000_b3": _md(4, 256, 33, 1000, 0, 3, "one slab per n-tile: the ring runs four n-tiles ahead"),
    "s1_nb512_k96_f1000": _md(1, 512, 96, 1000, 4, 1, "S = 1, three slabs per n-tile"),
    "s3_nb128_k128_f3999_b3": _md(3, 128, 128, 3999, 0, 3, "S = 3 of one n-tile each, long"),
    "s2_nb256_k129_refused": _md(2, 256, 129, 129, 4, 1, "K = 129 > the resident limit: refused", refuse=True),
}


@pytest.mark.parametrize("name", list(ROWS))
def test_maskdec_vs_fp64(name):
    r = ROWS[name]
    c = PW._case(name, r)
    st, out = PW._run(c, r, "f16x3")
    if r.get("refuse"):
        assert st == N.CTN_EUNSUPPORTED, f"{name}: status {st}, expected CTN_EUNSUPPORTED"
        assert bool((out["D"] == 0).all()), f"{name}: a refused call wrote its output"
        return
    assert st == N.CTN_OK, f"{name}: status {st}"
    res = PW._check(name, c, r, "f16x3", out)
    st2, out2 = PW._run(c, r, "f16x3")
    assert st2 == N.CTN_OK and torch.equal(out2["D"], out["D"]), f"{name}: second call differs"
    print(f"{name} [{r['reaches']}] e/bound " + " ".join(f"{k} {v:.3f}" for k, v in res.items()))


@pytest.mark.parametrize("skip,S", [(128, 2), (64, 3), (160, 2)])
def test_fused_forward_matches_unfused(skip, S):
    """forward (fused when K = skip <= 128) against extract_latent (always the unfused mask + decoder, another summation order)
    and against the CPU oracle"""
    from ctn_b200.models.conv_tasnet import ConvTasNet
    cfg = O.OracleConfig(n_basis=128, kernel_size=16, sep_hidden_channels=128, sep_bottleneck_channels=64, sep_skip_channels=skip,
                         sep_num_blocks=2, sep_num_layers=3, causal=False, n_sources=S)
    sd = O.synth_state_dict(cfg, seed=skip + S)
    m = ConvTasNet(cfg.n_basis, cfg.kernel_size, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None,
                   sep_hidden_channels=cfg.sep_hidden_channels, sep_bottleneck_channels=cfg.sep_bottleneck_channels,
                   sep_skip_channels=skip, sep_num_blocks=cfg.sep_num_blocks, sep_num_layers=cfg.sep_num_layers, causal=False,
                   n_sources=S)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    m.math = "f16x3"
    mixture, _ = O.synth_batch(3, S, 8003, seed=5)
    with torch.no_grad():
        fused = m(mixture.cuda())
        unfused, _ = m.extract_latent(mixture.cuda())
        again = m(mixture.cuda())
        ref, _ = O.conv_tasnet_fwd(mixture, sd, cfg)
    torch.testing.assert_close(fused, unfused, rtol=1e-4, atol=2e-5)
    assert torch.equal(fused, again), "a repeated forward differs"
    err = float((fused.cpu() - ref).abs().max())
    assert err < 2e-5 + 1e-4 * float(ref.abs().max()), f"skip {skip}, S {S}: max |out - oracle| = {err:.2e}"
