"""pw1 on its resident-operand kernel (k_pw1_resident: ctn_pw(..., PRO_NONE or PRO_RES, EPI_H, f16x3) with K <= 128) at the
shapes where it can go wrong (``-m gpu``).

Each row goes through the verification hook with the harness of test_pw_contraction_gpu.py, writes into NaN-filled outputs and
holds h, x_new and the gLN statistics to the same fp64 gate (e <= E_drop / 8).  Each call must be exactly one launch besides the
weight-image build, of the kernel the routing names: k_pw1_resident up to K = 128, k_pw_wgmma's channel-split tile at K = 129.
A second call gives h and x_new bit for bit (the statistics are double sums whose order is not fixed).
"""
import pytest
import torch

import test_pw_contraction_gpu as PW
from ctn_b200 import _native as N

pytestmark = pytest.mark.gpu

RESIDENT, SPLIT = "k_pw1_resident", "k_pw_wgmma"


def _r(pro, M, K, frames, reaches, B=1, **kw):
    return PW._row(pro, "h", M, K, frames, reaches, B=B, modes=["f16x3"], **kw)


ROWS = {
    "res_k128_m512_f3999_b2": _r("res", 512, 128, 3999, "the cfg2 pw1 shape (two samples): K at the routing limit", B=2),
    "res_k129_m512_f1000": _r("res", 512, 129, 1000, "K = 129: one past the limit, the channel-split tile of k_pw_wgmma"),
    "none_k128_m512_f65": _r("none", 512, 128, 65, "block 0 (PRO_NONE), one frame into the second tile"),
    "none_k129_m512_f64": _r("none", 512, 129, 64, "PRO_NONE at K = 129: k_pw_wgmma, one full tile"),
    "res_k100_m300_f63": _r("res", 300, 100, 63, "K = 100: a partial last slab; M = 300: the second warpgroup idle in pass 1"),
    "res_k64_m2048_f64": _r("res", 2048, 64, 64, "M = 2048: eight passes through each warpgroup's ring, two slabs per pass"),
    "none_k128_m300_f1_b3": _r("none", 300, 128, 1, "one frame, an idle warpgroup in the last pass", B=3),
    "res_k128_m512_f129_b37": _r("res", 512, 128, 129, "B = 37", B=37),
    "res_pre_k128_m512_f1000": _r("res", 512, 128, 1000, "store_pre with PRO_RES (the training forward)", store_pre=True),
    "none_pre_k33_m129_f3999": _r("none", 129, 33, 3999, "store_pre, a 1-channel last slab, a 1-row last n-tile", store_pre=True),
}


def _profiled_run(c, r):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        st, out = PW._run(c, r, "f16x3")
    # the library's launches: not the weight-image build, and not the NaN / zero fills and copies of the harness's own tensors
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "build_wimg" not in e.name
             and "emcpy" not in e.name and "emset" not in e.name and "at::" not in e.name]
    return st, out, names


@pytest.mark.parametrize("name", list(ROWS))
def test_pw1_resident_vs_fp64(name):
    r = ROWS[name]
    c = PW._case(name, r)
    st, out, names = _profiled_run(c, r)
    assert st == N.CTN_OK, f"{name}: status {st}"
    want = RESIDENT if r["K"] <= 128 else SPLIT
    assert len(names) == 1 and want in names[0], f"{name}: launches {names}, expected one {want}"
    res = PW._check(name, c, r, "f16x3", out)
    st2, out2 = PW._run(c, r, "f16x3")
    assert st2 == N.CTN_OK, f"{name}: second call status {st2}"
    assert torch.equal(out2["D"], out["D"]), f"{name}: second call differs in h"
    if "xnew" in out:  # without the NaN guard row past the last channel
        assert torch.equal(out2["xnew"][:-1], out["xnew"][:-1]), f"{name}: second call differs in x_new"
    print(f"{name} [{r['reaches']}] {names[0].split('(')[0]} e/bound " + " ".join(f"{k} {v:.3f}" for k, v in res.items()))
