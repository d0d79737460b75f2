"""Which training step a ConvTasNet takes under autograd, without a GPU: for every combination of causal, mask, in_channels and
the three training switches, the exception `model(x)` raises on a CPU tensor.  A model outside every training step is refused
before the CUDA check; every other model reaches the CUDA check, where the CPU tensor is refused."""
import itertools

import pytest
import torch

from ctn_b200.models.conv_tasnet import ConvTasNet

REFUSALS = {
    "M": (NotImplementedError, "train natively only with model.multichannel_training = True"),
    "E": (NotImplementedError, "multichannel training is built for non-causal models with a sigmoid mask"),
    "S": (NotImplementedError, "softmax-mask training is built for non-causal monaural models"),
    "K": (NotImplementedError, "causal (cLN) models train natively only with model.causal_training = True"),
    "C": (RuntimeError, "runs on CUDA (sm_90a) tensors only"),  # a training step takes the model: the CUDA check refuses x
}
SWITCHES = list(itertools.product([False, True], repeat=3))  # (causal_training, multichannel_training, softmax_training)
# (causal, mask, in_channels): the refusal for each entry of SWITCHES, in order
OUTCOMES = {
    (False, "sigmoid", 1): "C C C C C C C C",
    (False, "sigmoid", 2): "M M C C M M C C",
    (False, "softmax", 1): "C C C C C C C C",
    (False, "softmax", 2): "M M E E M M E E",
    (True, "sigmoid", 1): "K K K K C C C C",
    (True, "sigmoid", 2): "M M E E M M E E",
    (True, "softmax", 1): "K S K S C S C S",
    (True, "softmax", 2): "M M E E M M E E",
}
ROWS = [(key, sw, code) for key, codes in OUTCOMES.items() for sw, code in zip(SWITCHES, codes.split())]


def _id(row):
    (causal, mask, cin), (ct, mt, st), _ = row
    return "{}-{}-cin{}-ct{}-mt{}-st{}".format("causal" if causal else "gln", mask, cin, int(ct), int(mt), int(st))


@pytest.mark.parametrize("row", ROWS, ids=[_id(r) for r in ROWS])
def test_training_step_refusals(row):
    (causal, mask, cin), switches, code = row
    torch.manual_seed(0)
    model = ConvTasNet(16, 4, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=16,
                       sep_bottleneck_channels=8, sep_skip_channels=8, sep_num_blocks=1, sep_num_layers=2, causal=causal, n_sources=2,
                       mask_nonlinear=mask, in_channels=cin)
    model.causal_training, model.multichannel_training, model.softmax_training = switches
    x = torch.randn(2, 1, 64) if cin == 1 else torch.randn(2, 1, cin, 64)
    exc, fragment = REFUSALS[code]
    with pytest.raises(exc) as info:
        model(x)
    assert type(info.value) is exc
    assert fragment in str(info.value)
