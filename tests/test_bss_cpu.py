"""BSS Eval without a GPU: the fp64 oracle against an independent formulation, the C ABI's refusals (each returns before any
CUDA call), the workspace size's independence of T, and the drop-in shims' fall-through to the reference's own modules."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import bss_ref as R
from ctn_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced: every call below is refused before it would be


# white references: 1e-8 dB.  Coloured ones: the normal equations square the condition number of the delayed-reference matrix,
# so the oracle's dense solve and the QR route part at about 1e-8 dB there; 1e-6 dB is still 100 times below the GPU bound.
@pytest.mark.parametrize("S,T,coloured,tol", [(1, 2000, False, 1e-8), (2, 3001, False, 1e-8), (3, 2500, False, 1e-8),
                                              (2, 2200, True, 1e-6)])
def test_oracle_matches_qr_projection(S, T, coloured, tol):
    refs, ests = R.make_item(np.random.default_rng(10 * S + T), S, T, coloured)
    a = R.tables(refs.astype(np.float64), ests.astype(np.float64), R.project_fft)
    b = R.tables(refs.astype(np.float64), ests.astype(np.float64), R.project_qr)
    for x, y in zip(a, b):
        finite = np.isfinite(y)
        assert np.array_equal(finite, np.isfinite(x))
        assert np.all(np.abs(x[finite] - y[finite]) <= tol)
    if S == 1:
        assert np.isinf(a[1]).all()  # P_all = P_j: no interference at all


def test_oracle_permutation_and_validation():
    refs, ests = R.make_item(np.random.default_rng(3), 3, 2000)
    sdr, sir, sar, perm = R.bss_eval_sources(refs, ests)
    sdr_t, sir_t, _ = R.tables(refs.astype(np.float64), ests.astype(np.float64))
    assert np.array_equal(sdr, sdr_t[perm, np.arange(3)]) and sorted(perm) == [0, 1, 2]
    _, _, _, ident = R.bss_eval_sources(refs, ests, compute_permutation=False)
    assert list(ident) == [0, 1, 2]
    silent = refs.copy()
    silent[1] = 0
    with pytest.raises(ValueError):
        R.bss_eval_sources(silent, ests)
    with pytest.raises(ValueError):
        R.bss_eval_sources(refs, silent)
    with pytest.raises(ValueError):
        R.bss_eval_sources(refs, ests[:2])


def _call(**kw):
    a = dict(ref=FAKE, est=FAKE, B=2, K=2, S=2, T=1000, perm_on=1, sdr=FAKE, sir=FAKE, sar=FAKE, perm=FAKE, status=FAKE, ws=FAKE,
             ws_bytes=1 << 40, stream=None)
    a.update(kw)
    return N.ctn_bss_eval_sources(*a.values())


def test_abi_rejections():
    for name in ("ctn_bss_workspace_bytes", "ctn_bss_eval_sources"):
        assert hasattr(N.lib, name) and name in N.EXPORTED
    for bad in (dict(ref=None), dict(est=None), dict(sdr=None), dict(sir=None), dict(sar=None), dict(perm=None), dict(status=None),
                dict(ws=None), dict(B=0), dict(K=0), dict(S=0), dict(T=0), dict(S=-1), dict(T=-5)):
        assert _call(**bad) == N.CTN_EINVAL, bad
    assert _call(S=5) == N.CTN_EUNSUPPORTED
    assert _call(B=65536, K=1, S=1) == N.CTN_EUNSUPPORTED  # estimates ride on gridDim.y
    assert _call(ws=FAKE + 8) == N.CTN_EALIGN
    assert _call(ws_bytes=1024) == N.CTN_EWORKSPACE
    n = C.c_size_t(0)
    assert N.ctn_bss_workspace_bytes(1, 1, 5, 100, C.byref(n)) == N.CTN_EUNSUPPORTED
    assert N.ctn_bss_workspace_bytes(1, 1, 2, 0, C.byref(n)) == N.CTN_EINVAL
    assert N.ctn_bss_workspace_bytes(1, 1, 2, 100, None) == N.CTN_EINVAL


@pytest.mark.parametrize("B,K,S", [(1, 1, 1), (1, 2, 2), (5, 2, 3), (64, 2, 4)])
def test_workspace_does_not_grow_with_T(B, K, S):
    sizes = []
    for T in (1000, 1000000):
        n = C.c_size_t(0)
        assert N.ctn_bss_workspace_bytes(B, K, S, T, C.byref(n)) == N.CTN_OK
        sizes.append(n.value)
    assert sizes[0] == sizes[1]
    # the Gram matrix, its S diagonal blocks and their tile inverses dominate: B ((S L)^2 + S L^2) doubles and a little more
    floor = 8 * B * ((S * 512) ** 2 + S * 512 ** 2)
    assert floor < sizes[0] < 2 * floor + (64 << 20)


def test_python_rejects_on_the_host():
    import torch
    from ctn_b200.utils.bss import bss_eval_sources, bss_eval_sources_batch
    with pytest.raises(ValueError):
        bss_eval_sources(torch.ones(2, 100), torch.ones(3, 100))
    with pytest.raises(ValueError):
        bss_eval_sources_batch(torch.ones(1, 2, 100), torch.ones(1, 2, 2, 99))
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            bss_eval_sources(torch.ones(2, 100), torch.ones(2, 100))


def test_shims_fall_through_to_the_reference(tmp_path):
    """With PYTHONPATH = shim directory, then a reference src/ tree: what the shim provides is ours, the rest is the reference's"""
    for rel in ("utils/__init__.py", "criterion/__init__.py", "models/__init__.py", "modules/__init__.py"):
        (tmp_path / rel).parent.mkdir(parents=True, exist_ok=True)
        (tmp_path / rel).write_text("")
    (tmp_path / "utils" / "utils.py").write_text("def draw_loss_curve(*a, **k):\n    return 'fake-ref'\n")
    (tmp_path / "utils" / "bss.py").write_text("raise ImportError('the reference bss.py needs mir_eval')\n")
    (tmp_path / "criterion" / "distance.py").write_text("WHERE = 'fake-ref'\n")
    (tmp_path / "models" / "conv_tasnet.py").write_text("raise ImportError('shadowed by the shim')\n")
    pkg = os.path.join(ROOT, "dnn-based_source_separation_b200")
    code = ("import warnings; warnings.simplefilter('ignore');"
            "from utils.utils import draw_loss_curve; from utils.bss import bss_eval_sources; import criterion.distance as d;"
            "from models.conv_tasnet import ConvTasNet; import ctn_b200.models.conv_tasnet as m; import ctn_b200.utils.bss as b;"
            "import utils.utils as uu;"
            "assert draw_loss_curve() == 'fake-ref' and d.WHERE == 'fake-ref' and uu.__file__.startswith(%r);"
            "assert bss_eval_sources is b.bss_eval_sources and ConvTasNet is m.ConvTasNet;"
            "print('ok')" % str(tmp_path))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([pkg, str(tmp_path)]))
    out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr
