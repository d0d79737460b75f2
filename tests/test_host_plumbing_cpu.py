"""Host plumbing shared by the pipelines, without a GPU: one config check behind every entry point (the status of each
single-fault config), the workspace / state sizes the carves produce, and the ctn_params_t the Python side builds.
Every C call below is refused or answered before it would touch the device."""
import ctypes as C

import pytest
import torch

from ctn_b200 import _native as N
from ctn_b200.models import _train
from ctn_b200.models.conv_tasnet import ConvTasNet

FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced
OK, EINVAL, EUNSUP, EWS = N.CTN_OK, N.CTN_EINVAL, N.CTN_EUNSUPPORTED, N.CTN_EWORKSPACE

TINY = dict(n_basis=64, kernel_size=16, stride=8, bottleneck=32, hidden=64, skip=32, sep_kernel=3, num_blocks=2, num_layers=4, n_sources=2)
PAPER = dict(n_basis=512, kernel_size=16, stride=8, bottleneck=128, hidden=512, skip=128, sep_kernel=3, num_blocks=3, num_layers=8,
             n_sources=2)


def _cfg(base=TINY, **kw):
    c = N.Config()
    fields = dict(base, causal=0, enc_relu=0, mask_softmax=0, math=N.MATH_FP32, eps=1e-8, eps_tcn=1e-8, in_channels=1)
    fields.update(kw)
    for k, v in fields.items():
        setattr(c, k, v)
    return c


def _query(fn, cfg, *args):
    n = C.c_size_t(0)
    return fn(C.byref(cfg), *args, C.byref(n)), n.value


def _statuses(kw):
    """(model, TCN, training, online) status of a config; the online entry sees it on a causal base unless kw sets causal"""
    c = _cfg(**kw)
    return (_query(N.ctn_workspace_bytes, c, 2, 4000)[0], _query(N.ctn_tcn_workspace_bytes, c, 2, 500)[0],
            _query(N.ctn_train_workspace_bytes, c, 2, 4000)[0], _query(N.ctn_online_state_bytes, _cfg(**dict(dict(causal=1), **kw)), 2, 32)[0])


# EINVAL: a value no pipeline accepts; EUNSUPPORTED: a valid value outside one pipeline's envelope.  The TCN-only query ignores
# the encoder / mask / decoder fields.
SINGLE_FAULTS = [
    (dict(), (OK, OK, OK, OK)),
    (dict(n_basis=0), (EINVAL, OK, EINVAL, EINVAL)),
    (dict(kernel_size=0), (EINVAL, OK, EINVAL, EINVAL)),
    (dict(stride=0), (EINVAL, OK, EINVAL, EINVAL)),
    (dict(n_sources=0), (EINVAL, OK, EINVAL, EINVAL)),
    (dict(bottleneck=0), (EINVAL, EINVAL, EINVAL, EINVAL)),
    (dict(hidden=0), (EINVAL, EINVAL, EINVAL, EINVAL)),
    (dict(skip=0), (EINVAL, EINVAL, EINVAL, EINVAL)),
    (dict(sep_kernel=0), (EINVAL, EINVAL, EINVAL, EINVAL)),
    (dict(num_blocks=0), (EINVAL, EINVAL, EINVAL, EINVAL)),
    (dict(num_layers=0), (EINVAL, EINVAL, EINVAL, EINVAL)),
    (dict(kernel_size=12), (EINVAL, OK, EINVAL, EINVAL)),  # kernel_size % stride != 0
    (dict(math=7), (EINVAL, EINVAL, EINVAL, EINVAL)),
    (dict(mask_softmax=1), (OK, OK, EUNSUP, OK)),
    (dict(mask_softmax=2), (EINVAL, OK, EINVAL, EINVAL)),
    (dict(in_channels=-1), (EINVAL, OK, EINVAL, EINVAL)),
    (dict(in_channels=2), (OK, OK, EUNSUP, EUNSUP)),
    (dict(in_channels=100), (EINVAL, OK, EINVAL, EUNSUP)),  # online refuses multichannel before it checks the fields
    (dict(causal=1), (OK, OK, EUNSUP, OK)),
    (dict(causal=0), (OK, OK, OK, EUNSUP)),
    (dict(num_layers=21), (EUNSUP, EUNSUP, EUNSUP, EUNSUP)),
    (dict(num_blocks=9, num_layers=8), (EUNSUP, EUNSUP, EUNSUP, EUNSUP)),  # R*X = 72 > 64 blocks
]


@pytest.mark.parametrize("kw,expected", SINGLE_FAULTS, ids=[",".join(f"{k}={v}" for k, v in kw.items()) or "valid" for kw, _ in SINGLE_FAULTS])
def test_single_fault_status(kw, expected):
    assert _statuses(kw) == expected


def _blocks_fwd(n_blocks, **kw):
    blocks = (N.BlockParams * 65)()
    for b in blocks:
        for name in N.BLOCK_FIELDS:
            setattr(b, name, FAKE)
    dil = (C.c_int * 65)(*([1] * 65))
    return N.ctn_tcn_blocks_fwd(C.byref(_cfg(**kw)), blocks, n_blocks, dil, FAKE, None, FAKE, 1, 32, FAKE, 0, None)


@pytest.mark.parametrize("n_blocks,status", [(21, EWS), (64, EWS), (0, EINVAL), (65, EINVAL)])
def test_blocks_fwd_takes_up_to_64_blocks(n_blocks, status):
    """explicit dilations: any run of 1..64 blocks passes every config check (the empty workspace is what it refuses)"""
    assert _blocks_fwd(n_blocks) == status


def test_blocks_fwd_checks_the_config():
    assert _blocks_fwd(4, hidden=0) == EINVAL
    assert _blocks_fwd(4, math=7) == EINVAL
    assert _blocks_fwd(4, causal=1) == EUNSUP


# bytes at B = 2 (T = 32000 samples for the model / training workspaces, 4000 frames for the TCN, 64-frame chunks online)
BYTES = {
    ("paper", 0, N.MATH_FP32): dict(ws=311111936, tcn=260516352, train=1163137024),
    ("paper", 0, N.MATH_F16X3): dict(ws=350524672, tcn=298351104, train=1416402176),
    ("paper", 1, N.MATH_FP32): dict(ws=118830080, tcn=68234496, online=22563584, train=1172096736),
    ("paper", 1, N.MATH_F16X3): dict(ws=159292416, tcn=107118848, online=61976320, train=1173149408),
    ("tiny", 0, N.MATH_FP32): dict(ws=30572800, tcn=24272128, train=78686464),
    ("tiny", 0, N.MATH_F16X3): dict(ws=31471360, tcn=25070848, train=96548608),
    ("tiny", 1, N.MATH_FP32): dict(ws=16040960, tcn=9740288, online=692992, train=82526176),
    ("tiny", 1, N.MATH_F16X3): dict(ws=17005568, tcn=10605056, online=1591552, train=82657760),
}


@pytest.mark.parametrize("key", list(BYTES), ids=[f"{n}-{'causal' if c else 'gln'}-math{m}" for n, c, m in BYTES])
def test_workspace_bytes(key):
    name, causal, math = key
    base = PAPER if name == "paper" else TINY
    c = _cfg(base, causal=causal, math=math)
    got = dict(ws=_query(N.ctn_workspace_bytes, c, 2, 32000), tcn=_query(N.ctn_tcn_workspace_bytes, c, 2, 4000))
    if causal:
        got["online"] = _query(N.ctn_online_state_bytes, c, 2, 64)
        got["train"] = _query(N.ctn_causal_train_workspace_bytes, c, 2, 32000)
        # the causal step runs its contractions on tf32 pieces in the fp16-piece mode: the same workspace as tf32x3
        if math == N.MATH_F16X3:
            assert got["train"] == _query(N.ctn_causal_train_workspace_bytes, _cfg(base, causal=1, math=N.MATH_TF32X3), 2, 32000)
    else:
        got["train"] = _query(N.ctn_train_workspace_bytes, c, 2, 32000)
    for what, want in BYTES[key].items():
        status, n = got[what]
        assert status == OK
        assert want - 256 < n <= want, (what, n, want)  # a reordered carve may only save alignment padding


def _tiny_model():
    torch.manual_seed(0)
    m = ConvTasNet(64, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=64,
                   sep_bottleneck_channels=32, sep_skip_channels=32, sep_num_blocks=2, sep_num_layers=3, causal=False, n_sources=2)
    return m


def _check_struct(p, slots):
    n_blocks = 1 + max(s[0] for s, _ in slots if isinstance(s, tuple))
    for slot, t in slots:
        got = getattr(p.blocks[slot[0]], slot[1]) if isinstance(slot, tuple) else getattr(p, slot)
        assert got == (None if t is None else t.data_ptr()), slot
    assert [s for s, t in slots if t is None] == [(n_blocks - 1, "out_w"), (n_blocks - 1, "out_b")]


def test_model_params_point_at_the_tensors():
    m = _tiny_model()
    p, keep = m.native_params(torch.device("cpu"))
    _check_struct(p, _train.param_list(m))


def _training_struct(slots, dev):
    """the builder the training node calls for its parameters and their gradient views"""
    if not hasattr(N, "build_params"):  # a tree whose training node builds its structs itself
        return _train._struct([s for s, _ in slots], [t for _, t in slots], 1 + max(s[0] for s, _ in slots if isinstance(s, tuple)), dev)
    return N.build_params(slots, dev)


def test_training_params_point_at_the_tensors():
    m = _tiny_model()
    slots = _train.param_list(m)
    p, keep = _training_struct(slots, torch.device("cpu"))
    _check_struct(p, slots)
    # gradient views of one flat buffer, as the backward builds them
    flat = torch.zeros(sum(t.numel() for _, t in slots if t is not None))
    views, o = [], 0
    for s, t in slots:
        views.append((s, None if t is None else flat[o:o + t.numel()].view(t.shape)))
        o += 0 if t is None else t.numel()
    g, keep2 = _training_struct(views, torch.device("cpu"))
    _check_struct(g, views)


def test_params_refuse_a_foreign_tensor():
    m = _tiny_model().double()
    with pytest.raises(RuntimeError):
        m.native_params(torch.device("cpu"))
