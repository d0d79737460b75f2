"""ORPIT / Sinkhorn PIT without a GPU: the oracle's ``orpit`` / ``sinkpit`` against outputs of the unmodified reference
(tests/golden/pit_variants.pt, minted by ``tests/golden/make_pit_variants.py``), the drop-in shim's imports, and the C ABI's argument
rejections, which return before any CUDA call."""
import os

import pytest
import torch

import pit_variants_oracle as PO
from ctn_b200 import _native as N

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pit_variants.pt"))


def _close(a, b, rtol, what):
    err = float((a - b).abs().max())
    assert err <= rtol * float(b.abs().max()) + 1e-7, f"{what}: max|diff| {err:.3e} vs scale {float(b.abs().max()):.3e}"


@pytest.mark.parametrize("k", range(len(GOLD["orpit"])), ids=[f"{r['name']}-{r['criterion']}" for r in GOLD["orpit"]])
def test_oracle_orpit_matches_reference(k):
    r = GOLD["orpit"][k]
    maximize = r["criterion"] == "SISDR"
    x = r["input"].clone().requires_grad_(True)
    loss, idx = PO.orpit(x, r["target"], r["lengths"], maximize=maximize, batch_mean=True)
    loss.backward()
    loss_b, _ = PO.orpit(r["input"], r["target"], r["lengths"], maximize=maximize, batch_mean=False)
    assert abs(float(loss.detach()) - float(r["loss"])) <= 1e-5
    assert float((loss_b - r["loss_b"]).abs().max()) <= 1e-5
    assert torch.equal(idx, r["indices"])
    assert torch.equal(r["patterns"], torch.tensor([[0, 1], [1, 0]]))
    _close(x.grad, r["grad"], 1e-5, "input gradient")


@pytest.mark.parametrize("k", range(len(GOLD["sinkpit"])),
                         ids=[f"S{r['S']}-K{r['K']}-c{r['coldness']:g}-{r['criterion']}" for r in GOLD["sinkpit"]])
def test_oracle_sinkpit_matches_reference(k):
    r = GOLD["sinkpit"][k]
    inp = GOLD["sinkpit_inputs"][r["S"]]
    x = inp["input"].clone().requires_grad_(True)
    loss, P = PO.sinkpit(x, inp["target"], coldness=r["coldness"], iteration=r["K"], maximize=r["criterion"] == "SISDR")
    loss.backward()
    assert abs(float(loss.detach()) - float(r["loss"])) <= 1e-5 * max(1.0, abs(float(r["loss"])))
    assert float((P.detach() - r["P"]).abs().max()) <= 1e-5
    assert torch.equal(torch.argmax(P.detach(), dim=2), r["pattern"])
    _close(x.grad, r["grad"], 1e-5, "input gradient")


def test_shim_exports_the_new_criteria():
    from criterion.pit import ORPIT, sinkpit, SinkPIT  # noqa: F401  (the recipes' imports)
    from ctn_b200.criterion.pit import ORPIT as A, sinkpit as B, SinkPIT as C
    assert (ORPIT, sinkpit, SinkPIT) == (A, B, C)
    from ctn_b200.criterion.sdr import NegSISDR
    assert torch.equal(ORPIT(NegSISDR()).patterns, torch.tensor([[0, 1], [1, 0]]))


def test_orpit_rejects_a_single_target():
    """n_b = 1 raises ValueError before any computation (the reference divides by n_b - 1 = 0)"""
    from ctn_b200.criterion.pit import ORPIT
    from ctn_b200.criterion.sdr import NegSISDR
    r = GOLD["orpit"][2]
    with pytest.raises(ValueError):
        ORPIT(NegSISDR())(r["input"][:1], r["target"][:1, :1])
    packed = torch.nn.utils.rnn.pack_sequence([r["target"][0, :3], r["target"][1, :1]], enforce_sorted=False)
    with pytest.raises(ValueError):
        ORPIT(NegSISDR())(r["input"][:2], packed)


FAKE = 1 << 20  # a non-null pointer that is never dereferenced: every call below is rejected before any CUDA call


def test_orpit_abi_rejections():
    assert N.ctn_orpit_scratch_bytes(0, 3) == 0
    assert N.ctn_orpit_scratch_bytes(2, 3) == 8 * 2 * (2 * 6 + 6) + 4 * 2 * (2 * 3 + 2)
    args = lambda **kw: {**dict(est=FAKE, tgt=FAKE, n_b=None, B=2, n=3, T=100, eps=1e-8, maximize=0, loss_b=FAKE, idx=FAKE,
                                scratch=FAKE, stream=None), **kw}
    fwd = lambda a: N.ctn_orpit_fwd(*a.values())
    for bad in (dict(est=None), dict(tgt=None), dict(loss_b=None), dict(idx=None), dict(scratch=None), dict(B=0), dict(T=0),
                dict(n=1)):
        assert fwd(args(**bad)) == N.CTN_EINVAL, bad
    assert fwd(args(n=17)) == N.CTN_EUNSUPPORTED
    bwd = lambda **kw: N.ctn_orpit_bwd(*{**dict(est=FAKE, tgt=FAKE, n_b=None, idx=FAKE, B=2, n=3, T=100, eps=1e-8, maximize=0,
                                                scratch=FAKE, g=None, d=FAKE, stream=None), **kw}.values())
    for bad in (dict(idx=None), dict(d=None), dict(est=None), dict(n=1)):
        assert bwd(**bad) == N.CTN_EINVAL, bad
    assert bwd(n=17) == N.CTN_EUNSUPPORTED


def test_sinkpit_abi_rejections():
    assert N.ctn_sinkpit_scratch_bytes(2, 3, -1) == 0
    assert N.ctn_sinkpit_scratch_bytes(2, 3, 10) == 8 * 2 * (2 * 9 + 3 + 9 + 2 * 10 * 3) + 4 * 2 * (9 + 3)
    fwd = lambda **kw: N.ctn_sinkpit_fwd(*{**dict(est=FAKE, tgt=FAKE, B=2, S=3, T=100, K=10, c=1.0, eps=1e-8, maximize=0,
                                                  loss_b=FAKE, P=FAKE, pair=None, scratch=FAKE, stream=None), **kw}.values())
    for bad in (dict(est=None), dict(tgt=None), dict(loss_b=None), dict(P=None), dict(scratch=None), dict(B=0), dict(T=0),
                dict(S=0), dict(K=-1), dict(c=0.0), dict(c=-1.0), dict(c=float("inf")), dict(c=float("nan"))):
        assert fwd(**bad) == N.CTN_EINVAL, bad
    assert fwd(S=17) == N.CTN_EUNSUPPORTED
    bwd = lambda **kw: N.ctn_sinkpit_bwd(*{**dict(est=FAKE, tgt=FAKE, B=2, S=3, T=100, K=10, c=1.0, eps=1e-8, maximize=0,
                                                  scratch=FAKE, g=None, gP=None, dL=FAKE, d=FAKE, stream=None), **kw}.values())
    for bad in (dict(dL=None), dict(d=None), dict(scratch=None), dict(K=-1)):
        assert bwd(**bad) == N.CTN_EINVAL, bad
    assert bwd(S=17) == N.CTN_EUNSUPPORTED
