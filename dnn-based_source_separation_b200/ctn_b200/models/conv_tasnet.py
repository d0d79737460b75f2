"""Conv-TasNet on hand-written sm_90a kernels, behind the reference's class API.

Mirrors src/models/conv_tasnet.py of the reference: ``ConvTasNet`` (:16-320; constructor :57-66, forward :116-119,
extract_latent :121-171, get_config :173-198, build_model :199-236) and ``Separator`` (:322-378).  Module tree and
``state_dict`` keys are identical, so reference checkpoints load with ``load_state_dict``.

One forward is one C call (ctn_convtasnet_fwd, include/ctn_b200.h): encoder (+gLN statistics) -> gLN folded into the
bottleneck 1x1 -> R*X fused residual blocks -> PReLU + mask 1x1 + sigmoid + (w * mask) -> transposed-conv decoder with
the crop fused.  Internally activations are (batch, channels, pitch) fp32 with pitch = frames rounded up to 128.

Kernel envelope (anything else raises NotImplementedError, there is no eager fallback): enc_basis = dec_basis =
'trainable', in_channels = 1, 3-D input, dilated, separable, sep_nonlinear='prelu', sep_norm, mask_nonlinear='sigmoid'.
causal=False (gLN) runs the fused stack; causal=True (cLN) an un-fused pipeline (csrc/ctn_causal.cu), which trains natively
once ``model.causal_training = True`` is set.  Multichannel models (in_channels = C > 1, the 4-D input (B, 1, C, T) of the MUSDB18
recipes) train natively once ``model.multichannel_training = True`` is set (non-causal, sigmoid mask).  Softmax-mask models
(mask_nonlinear='softmax', the ORPIT and Sinkhorn PIT recipes) run forward in every configuration and train natively once
``model.softmax_training = True`` is set (non-causal, monaural); that step also returns the gradient w.r.t. a mixture that
requires grad, which the ORPIT recipe's recursive fine-tune step needs.
"""
import ctypes as C

import torch
import torch.nn as nn

from .. import _native as N
from ..utils.filterbank import choose_filterbank
from ..utils.tasnet import choose_layer_norm
from . import tdcn as _tdcn
from .tdcn import TimeDilatedConvNet, block_slots, resolve_math

EPS = 1e-12
DEFAULT_MATH = None
# separate_track's default segments per forward: one batch of model workspace stays under about 8 GB at the MUSDB18 recipe's size
# (ctn_separate_track_workspace_bytes; see the method's docstring)
TRACK_CHUNK_BATCH = 3


def _load_checkpoint(path):
    """trainer checkpoints are plain dicts of tensors / python scalars: try the safe loader first"""
    try:
        return torch.load(path, map_location="cpu", weights_only=True)
    except Exception:
        return torch.load(path, map_location="cpu", weights_only=False)


class Separator(nn.Module):
    def __init__(self, num_features, bottleneck_channels=128, hidden_channels=256, skip_channels=128, kernel_size=3,
                 num_blocks=3, num_layers=8, dilated=True, separable=True, causal=True, nonlinear='prelu', norm=True,
                 mask_nonlinear='sigmoid', n_sources=2, eps=EPS):
        super().__init__()
        self.num_features, self.n_sources, self.eps, self.causal = num_features, n_sources, eps, causal
        self.norm1d = choose_layer_norm('cLN' if causal else 'gLN', num_features, causal=causal, eps=eps)
        self.bottleneck_conv1d = nn.Conv1d(num_features, bottleneck_channels, kernel_size=1, stride=1)
        # the reference builds the TDCN without forwarding eps (conv_tasnet.py:336-339) -> default 1e-12
        self.tdcn = TimeDilatedConvNet(bottleneck_channels, hidden_channels=hidden_channels, skip_channels=skip_channels,
                                       kernel_size=kernel_size, num_blocks=num_blocks, num_layers=num_layers, dilated=dilated,
                                       separable=separable, causal=causal, nonlinear=nonlinear, norm=norm)
        self.prelu = nn.PReLU()
        self.mask_conv1d = nn.Conv1d(skip_channels, n_sources * num_features, kernel_size=1, stride=1)
        if mask_nonlinear == 'sigmoid':
            self.mask_softmax = False
        elif mask_nonlinear == 'softmax':
            self.mask_softmax = True   # nn.Softmax(dim=1) over ALL n_sources*num_features channels (conv_tasnet.py:345-357); trains with ConvTasNet.softmax_training
        else:
            raise ValueError("Cannot support {}".format(mask_nonlinear))
        self.math = None

    # ---- native plumbing -------------------------------------------------------------------------
    def native_config(self, kernel_size=1, stride=1, enc_relu=False):
        mode = self.math if self.math is not None else (DEFAULT_MATH if DEFAULT_MATH is not None else _tdcn.DEFAULT_MATH)  # DEFAULT_MATH here: legacy override
        cfg = self.tdcn.native_config(n_basis=self.num_features, kernel_size=kernel_size, stride=stride,
                                      n_sources=self.n_sources, enc_relu=int(enc_relu), mask_softmax=int(self.mask_softmax))
        cfg.math = resolve_math(mode)
        cfg.eps = float(self.eps)
        return cfg

    def param_slots(self, enc_w=None, dec_w=None):
        """[(slot, tensor-or-None)] in the order of ctn_params_t: slot = top-level field name or (block index, block field name)"""
        g0, b0 = N.norm_affine(self.norm1d)
        top = dict(enc_w=enc_w, norm0_g=g0, norm0_b=b0, bn_w=self.bottleneck_conv1d.weight, bn_b=self.bottleneck_conv1d.bias,
                   prelu_out=self.prelu.weight, mask_w=self.mask_conv1d.weight, mask_b=self.mask_conv1d.bias, dec_w=dec_w)
        return [(k, top[k]) for k in N.TOP_FIELDS] + block_slots(self.tdcn.residual_blocks())

    def native_params(self, dev, enc_w=None, dec_w=None):
        return N.build_params(self.param_slots(enc_w, dec_w), dev)

    def forward(self, input):
        """input (batch_size, num_features, n_frames) -> mask (batch_size, n_sources, num_features, n_frames)"""
        if input.dim() != 3 or input.size(1) != self.num_features:
            raise ValueError("input.size() is expected (?, {}, ?), but given {}".format(self.num_features, tuple(input.size())))
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("stand-alone Separator.forward is inference-only (training runs through ConvTasNet.forward, one autograd node): call under torch.no_grad()")
        w = input.contiguous()
        dev = N.require_cuda(w)
        B, _, frames = w.shape
        cfg = self.native_config()
        params, keep = self.native_params(dev)
        need = C.c_size_t(0)
        N.check(N.ctn_workspace_bytes(C.byref(cfg), B, frames, C.byref(need)), "ctn_workspace_bytes")  # kernel 1, stride 1: T == frames
        pitch = N.ctn_pitch(frames)
        extra = 4 * B * self.n_sources * self.num_features * pitch + 1024
        base, nbytes = N.aligned(N.workspace(dev, need.value + extra))
        mask = torch.empty(B, self.n_sources, self.num_features, frames, dtype=torch.float32, device=dev)
        N.check(N.ctn_separator_fwd(C.byref(cfg), C.byref(params), w.data_ptr(), B, frames, mask.data_ptr(), base, nbytes,
                                    N.stream_ptr(dev)), "ctn_separator_fwd")
        return mask


class ConvTasNet(nn.Module):
    def __init__(self, n_basis, kernel_size, stride=None, enc_basis=None, dec_basis=None,
                 sep_hidden_channels=256, sep_bottleneck_channels=128, sep_skip_channels=128, sep_kernel_size=3,
                 sep_num_blocks=3, sep_num_layers=8, dilated=True, separable=True, sep_nonlinear='prelu', sep_norm=True,
                 mask_nonlinear='sigmoid', causal=True, n_sources=2, eps=EPS, **kwargs):
        super().__init__()
        if stride is None:
            stride = kernel_size // 2
        assert kernel_size % stride == 0, "kernel_size is expected divisible by stride"

        self.in_channels = kwargs.get('in_channels', 1)
        self.n_basis, self.kernel_size, self.stride = n_basis, kernel_size, stride
        self.enc_basis, self.dec_basis = enc_basis, dec_basis
        self.enc_nonlinear = kwargs['enc_nonlinear'] if (enc_basis == 'trainable' and dec_basis != 'pinv') else None
        self.window_fn, self.enc_onesided, self.enc_return_complex = None, None, None

        self.sep_hidden_channels, self.sep_bottleneck_channels = sep_hidden_channels, sep_bottleneck_channels
        self.sep_skip_channels, self.sep_kernel_size = sep_skip_channels, sep_kernel_size
        self.sep_num_blocks, self.sep_num_layers = sep_num_blocks, sep_num_layers
        self.dilated, self.separable, self.causal = dilated, separable, causal
        self.sep_nonlinear, self.sep_norm, self.mask_nonlinear = sep_nonlinear, sep_norm, mask_nonlinear
        self.n_sources, self.eps = n_sources, eps

        encoder, decoder = choose_filterbank(n_basis, kernel_size=kernel_size, stride=stride, enc_basis=enc_basis,
                                             dec_basis=dec_basis, **kwargs)
        self.encoder = encoder
        self.separator = Separator(n_basis, bottleneck_channels=sep_bottleneck_channels, hidden_channels=sep_hidden_channels,
                                   skip_channels=sep_skip_channels, kernel_size=sep_kernel_size, num_blocks=sep_num_blocks,
                                   num_layers=sep_num_layers, dilated=dilated, separable=separable, causal=causal,
                                   nonlinear=sep_nonlinear, norm=sep_norm, mask_nonlinear=mask_nonlinear, n_sources=n_sources,
                                   eps=eps)
        self.decoder = decoder
        self.math = None  # numeric mode override: 'fp32' | 'tf32x3' | 'tf32'
        # causal (cLN) models train through the native causal pipeline only when this is set; off, they refuse autograd as before
        self.causal_training = False
        # multichannel (in_channels > 1) models train through the native multichannel step only when this is set; off, they refuse
        # autograd as before
        self.multichannel_training = False
        # softmax-mask models train through the native softmax step only when this is set; off, they refuse autograd as before
        self.softmax_training = False
        self.last_launches = 0
        self.last_chunk_perms = None  # separate_long: the chunk permutations of the last call

    # ---- reference API ---------------------------------------------------------------------------
    def forward(self, input):
        output, _ = self._run(input, want_latent=False)
        return output

    def extract_latent(self, input):
        """input (batch_size, 1, T) -> output (batch_size, n_sources, T), latent (batch_size, n_sources, n_basis, T')"""
        return self._run(input, want_latent=True)

    def get_config(self):
        return {
            'in_channels': self.in_channels, 'n_basis': self.n_basis, 'kernel_size': self.kernel_size, 'stride': self.stride,
            'enc_basis': self.enc_basis, 'dec_basis': self.dec_basis, 'enc_nonlinear': self.enc_nonlinear,
            'window_fn': self.window_fn, 'enc_onesided': self.enc_onesided, 'enc_return_complex': self.enc_return_complex,
            'sep_hidden_channels': self.sep_hidden_channels, 'sep_bottleneck_channels': self.sep_bottleneck_channels,
            'sep_skip_channels': self.sep_skip_channels, 'sep_kernel_size': self.sep_kernel_size,
            'sep_num_blocks': self.sep_num_blocks, 'sep_num_layers': self.sep_num_layers,
            'dilated': self.dilated, 'separable': self.separable, 'causal': self.causal,
            'sep_nonlinear': self.sep_nonlinear, 'sep_norm': self.sep_norm, 'mask_nonlinear': self.mask_nonlinear,
            'n_sources': self.n_sources, 'eps': self.eps,
        }

    def get_package(self):
        return self.get_config()

    @classmethod
    def build_model(cls, model_path, load_state_dict=False):
        """Rebuild from a trainer checkpoint (dict = get_config() + 'state_dict'); tolerates the legacy keys
        n_bases / enc_bases / dec_bases like the reference (conv_tasnet.py:204-206)."""
        config = _load_checkpoint(model_path)
        get = config.get
        model = cls(
            get('n_bases') or config['n_basis'], in_channels=get('in_channels') or 1,
            kernel_size=config['kernel_size'], stride=config['stride'],
            enc_basis=get('enc_bases') or config['enc_basis'], dec_basis=get('dec_bases') or config['dec_basis'],
            enc_nonlinear=config['enc_nonlinear'], window_fn=config['window_fn'],
            enc_onesided=get('enc_onesided') or None, enc_return_complex=get('enc_return_complex') or None,
            sep_hidden_channels=config['sep_hidden_channels'], sep_bottleneck_channels=config['sep_bottleneck_channels'],
            sep_skip_channels=config['sep_skip_channels'], sep_kernel_size=config['sep_kernel_size'],
            sep_num_blocks=config['sep_num_blocks'], sep_num_layers=config['sep_num_layers'],
            dilated=config['dilated'], separable=config['separable'], causal=config['causal'],
            sep_nonlinear=config['sep_nonlinear'], sep_norm=config['sep_norm'], mask_nonlinear=config['mask_nonlinear'],
            n_sources=config['n_sources'], eps=config['eps'])
        if load_state_dict:
            model.load_state_dict(config['state_dict'])
        return model

    # Google-Drive ids of the reference's published checkpoints (conv_tasnet.py:17-55); the files themselves are fetched by the
    # reference's utils.utils.download_pretrained_model_from_google_drive -- this path only LOADS them (same directory layout)
    pretrained_model_ids = {
        "wsj0-mix": {8000: {2: {"enc_relu": "1yy-o7TyS1EcBWZ41rskMAVavtuEi4fMe"}, 3: {"enc_relu": "1-4Abl7LnEtwqMnAFQOcNLUOaDbgp3NoG"}},
                     16000: {2: "", 3: ""}},
        "wham/enhance-single": {8000: "1-6oiSK_CEE5Vl4OCy8TinA0cKsFFfGUg", 16000: ""},
        "wham/enhance-both": {8000: "1-GISUVcWjMeP3GLvojz9b0svw6gkmd2G", 16000: ""},
        "wham/separate-noisy": {8000: "1-0ckoPjaIiTJwv9Qotz6fkY2xeC77xdi", 16000: ""},
        "musdb18": {44100: {"4sec_L20": "1A6dIofHZJQCUkyq-vxZ6KbPmEHLcf4WK", "8sec_L20": "1C4uv2z0w1s4rudIMaErLyEccNprJQWSZ",
                            "8sec_L64": "1paXNGgH8m0kiJTQnn1WH-jEIurCKXwtw"}},
        "librispeech": {16000: {2: "1NI6Q_WZHiTKkgkNTEcZE1yHskHgYUHpy"}},
    }

    @classmethod
    def build_from_pretrained(cls, root="./pretrained", quiet=False, load_state_dict=True, **kwargs):
        """conv_tasnet.py:239-310: resolve <root>/ConvTasNet/<task>/sr.../model/<choice>.pth from (task, sample_rate, n_sources, config,
        model_choice) exactly like the reference and build the model from it.  The download step is the reference's own helper
        (Google Drive); when the file is not there and that helper is not importable, FileNotFoundError names the expected path."""
        import os
        task = kwargs.get('task')
        if task not in cls.pretrained_model_ids:
            raise KeyError("Invalid task ({}) is specified.".format(task))
        ids = cls.pretrained_model_ids[task]
        extra = {}
        if task in ['wsj0-mix', 'wsj0']:
            sample_rate = kwargs.get('sample_rate') or 8000
            n_sources = kwargs.get('n_sources') or 2
            config = kwargs.get('config') or 'enc_relu'
            model_id = ids[sample_rate][n_sources][config]
            download_dir = os.path.join(root, cls.__name__, task, "sr{}/{}speakers/{}".format(sample_rate, n_sources, config))
            extra['n_sources'] = n_sources
        elif task == 'musdb18':
            sample_rate = kwargs.get('sample_rate') or 44100
            config = kwargs.get('config') or '4sec_L20'
            model_id = ids[sample_rate][config]
            download_dir = os.path.join(root, cls.__name__, task, "sr{}".format(sample_rate), config)
        elif task in ['wham/separate-noisy', 'wham/enhance-single', 'wham/enhance-both']:
            sample_rate = kwargs.get('sample_rate') or 8000
            model_id = ids[sample_rate]
            download_dir = os.path.join(root, cls.__name__, task, "sr{}".format(sample_rate))
        elif task == 'librispeech':
            sample_rate = kwargs.get('sample_rate') or 16000
            n_sources = kwargs.get('n_sources') or 2
            model_id = ids[sample_rate][n_sources]
            download_dir = os.path.join(root, cls.__name__, task, "sr{}/{}speakers".format(sample_rate, n_sources))
            extra['n_sources'] = n_sources
        else:
            raise NotImplementedError("Not support task={}.".format(task))
        extra['sample_rate'] = sample_rate
        model_choice = kwargs.get('model_choice') or 'best'
        model_path = os.path.join(download_dir, "model", "{}.pth".format(model_choice))
        if not os.path.exists(model_path):
            try:
                from utils.utils import download_pretrained_model_from_google_drive  # the reference's helper, when src/ is on the path
            except Exception:
                raise FileNotFoundError("{} not found (Google-Drive id {!r}); place the reference checkpoint there -- this path loads "
                                        "checkpoints, it does not download them".format(model_path, model_id))
            download_pretrained_model_from_google_drive(model_id, download_dir, quiet=quiet)
        config = _load_checkpoint(model_path)
        model = cls.build_model(model_path, load_state_dict=load_state_dict)
        if task == 'musdb18':
            extra.update({'sources': config['sources'], 'n_sources': len(config['sources'])})
        for key, value in extra.items():
            setattr(model, key, value)
        return model

    def online(self, batch_size=1, max_chunk=256):
        """Online (chunk-by-chunk) separator of this causal model for ``batch_size`` concurrent streams, pushes of at most
        ``max_chunk`` samples (a multiple of the stride): see ``ctn_b200.models.online.OnlineSeparator``."""
        from .online import OnlineSeparator
        return OnlineSeparator(self, batch_size, max_chunk)

    def separate_long(self, mixture, chunk, hop=None, chunk_batch=16, align=True):
        """Separate recordings of any length: mixture (batch, 1, T) -> (batch, n_sources, T), inference only, one C call
        (ctn_convtasnet_separate_long) without a host synchronisation.  The signal is cut into chunks of ``chunk`` samples every
        ``hop`` (default chunk // 2; chunk // 2 <= hop <= chunk), the last one moved left to end at T; the chunks run through
        the forward ``chunk_batch`` at a time; with ``align`` (and n_sources > 1; needs hop < chunk, n_sources <= 6) each
        chunk's sources are put in the order of the chunk before it by the inner products over the samples they share; the
        chunks are cross-faded with sin^2 ramps.  T <= chunk gives ``self(mixture)``.  The permutations used are kept in
        ``last_chunk_perms`` (batch, n_chunks, n_sources) int32: row [b, k, s] of chunk k carries output source s."""
        if mixture.dim() != 3 or mixture.size(1) != 1:
            if mixture.dim() == 4:
                raise NotImplementedError("separate_long takes (batch, 1, T): multichannel input is not built (whole multichannel "
                                          "tracks separate through separate_track)")
            raise ValueError("mixture.size() is expected (?, 1, ?), but given {}".format(tuple(mixture.size())))
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("separate_long is inference-only: call it under torch.no_grad()")
        x = mixture.contiguous()
        dev = N.require_cuda(x)
        B, _, T = x.shape
        chunk, chunk_batch = int(chunk), int(chunk_batch)
        hop = chunk // 2 if hop is None else int(hop)
        K = N.ctn_chunk_plan(T, chunk, hop, None, 0)
        if K < 0:
            N.check(K, "ctn_chunk_plan(T={}, chunk={}, hop={})".format(T, chunk, hop))
        cfg = self.native_config()
        params, keep = self.native_params(dev)
        need = C.c_size_t(0)
        N.check(N.ctn_separate_long_workspace_bytes(C.byref(cfg), B, T, chunk, hop, chunk_batch, C.byref(need)),
                "ctn_separate_long_workspace_bytes")
        base, nbytes = N.aligned(N.workspace(dev, need.value, tag="separate_long"))
        out = torch.empty(B, self.n_sources, T, dtype=torch.float32, device=dev)
        perms = torch.empty(B, K, self.n_sources, dtype=torch.int32, device=dev)
        N.check(N.ctn_convtasnet_separate_long(C.byref(cfg), C.byref(params), x.data_ptr(), B, T, chunk, hop, chunk_batch, int(bool(align)),
                                               out.data_ptr(), perms.data_ptr(), base, nbytes, N.stream_ptr(dev)),
                "ctn_convtasnet_separate_long")
        self.last_launches = N.ctn_last_launch_count()
        self.last_chunk_perms = perms
        return out

    def separate_track(self, mixture, segment, hop=None, chunk_batch=TRACK_CHUNK_BATCH):
        """Separate whole tracks the way the MUSDB18 recipe's tester does, in one C call (ctn_convtasnet_separate_track) without a
        host synchronisation, inference only.  A multichannel model takes (batch, 1, n_mics, T) and returns (batch, n_sources,
        n_mics, T); a monaural one (batch, 1, T) -> (batch, n_sources, T).

        Every segment and channel is standardised on its own, (x - mean) / (std + eps) with the unbiased std and this model's
        ``eps``, run through the model, and mapped back with std * estimate + mean (the mixture's statistics for every source).
        ``hop=None`` is the tester's layout: the track is zero-padded to a multiple of ``segment`` (the zeros count in the
        statistics), cut into segments that share no samples, and the estimates are concatenated and cropped to T.
        ``segment // 2 <= hop <= segment`` instead cuts chunks every ``hop`` samples like ``separate_long`` (the last one moved
        left to end at T, nothing padded) and cross-fades them with sin^2 ramps.  There is no permutation alignment: stems
        have a fixed order.

        The segments run through the forward ``chunk_batch`` at a time.  The default, 3, keeps one batch of model workspace at
        7.9 GB (2.6 GB per segment) for the recipe's separator (N = 256, L = 20, H = 512, B = 256, Sc = 128, X = 10, R = 4,
        four stereo sources, f16x3) on 8 s segments at 44.1 kHz; the whole call then needs 8.2 GB of workspace for a 240 s track."""
        C_in = int(self.in_channels)
        n_dims = mixture.dim()
        if n_dims == 3:
            if mixture.size(1) != 1:
                raise ValueError("input.size() is expected (?, 1, ?), but given {}".format(tuple(mixture.size())))
            if C_in != 1:
                raise ValueError("a model with in_channels={} takes the 4-D input (batch, 1, n_mics, T)".format(C_in))
        elif n_dims == 4:
            if mixture.size(1) != 1:
                raise ValueError("input.size() is expected (?, 1, ?, ?), but given {}".format(tuple(mixture.size())))
            if mixture.size(2) != C_in:
                raise ValueError("n_mics={} does not match in_channels={}".format(mixture.size(2), C_in))
        else:
            raise ValueError("Not support {} dimension input".format(n_dims))
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("separate_track is inference-only: call it under torch.no_grad()")
        B, T = mixture.size(0), mixture.size(-1)
        x = mixture.reshape(B, C_in, T).contiguous()
        dev = N.require_cuda(x)
        segment, chunk_batch = int(segment), int(chunk_batch)
        hop = 0 if hop is None else int(hop)
        K = N.ctn_track_plan(T, segment, hop, None, 0)
        if K < 0:
            N.check(K, "ctn_track_plan(T={}, segment={}, hop={})".format(T, segment, hop))
        cfg = self.native_config()
        params, keep = self.native_params(dev)
        need = C.c_size_t(0)
        N.check(N.ctn_separate_track_workspace_bytes(C.byref(cfg), B, T, segment, hop, chunk_batch, C.byref(need)),
                "ctn_separate_track_workspace_bytes")
        base, nbytes = N.aligned(N.workspace(dev, need.value, tag="separate_track"))
        out = torch.empty((B, self.n_sources, C_in, T) if n_dims == 4 else (B, self.n_sources, T), dtype=torch.float32, device=dev)
        N.check(N.ctn_convtasnet_separate_track(C.byref(cfg), C.byref(params), x.data_ptr(), B, T, segment, hop, chunk_batch,
                                                out.data_ptr(), base, nbytes, N.stream_ptr(dev)),
                "ctn_convtasnet_separate_track")
        self.last_launches = N.ctn_last_launch_count()
        return out

    @property
    def num_parameters(self):
        return sum(p.numel() for p in self.parameters() if p.requires_grad)

    def separate_host(self, mixture_host, sources_host, out_host=None, loss_eps=EPS):
        """End-to-end call on HOST buffers (ctn_convtasnet_loss_host): H2D copies of the (pinned) mixture (B,1,T) and sources
        (B,S,T), forward + PIT(NegSISDR) on the device, D2H of the estimates into ``out_host`` (optional), the mean loss and the
        permutation -- all enqueued on the current stream.  Returns (loss (1,) pinned, perm (B,S) int64 pinned); the caller
        synchronises the stream before reading them."""
        dev = self.encoder.conv1d.weight.device
        if dev.type != "cuda":
            raise RuntimeError("ctn_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        B, _, T = mixture_host.shape
        key = (B, T, dev)
        st = getattr(self, "_host_state", None)
        if st is None or st[0] != key:
            loss = torch.empty(1, dtype=torch.float32).pin_memory()
            perm = torch.empty(B, self.n_sources, dtype=torch.int64).pin_memory()
            st = (key, loss, perm)
            self._host_state = st
        _, loss, perm = st
        cfg = self.native_config()
        params, keep = self.native_params(dev)
        need = C.c_size_t(0)
        N.check(N.ctn_workspace_bytes(C.byref(cfg), B, T, C.byref(need)), "ctn_workspace_bytes")
        wbase, wbytes = N.aligned(N.workspace(dev, need.value))
        io_bytes = N.ctn_host_io_bytes(C.byref(cfg), B, T)
        ibase, ibytes = N.aligned(N.workspace(dev, io_bytes + 256, tag="host_io"))
        with torch.cuda.device(dev):
            N.check(N.ctn_convtasnet_loss_host(C.byref(cfg), C.byref(params), mixture_host.data_ptr(), sources_host.data_ptr(), B, T,
                                               N.ptr(out_host), loss.data_ptr(), perm.data_ptr(), ibase, ibytes, wbase, wbytes,
                                               float(loss_eps), N.stream_ptr(dev)), "ctn_convtasnet_loss_host")
        self.last_launches = N.ctn_last_launch_count()
        return loss, perm

    # ---- native plumbing ---------------------------------------------------------------------------
    def native_config(self):
        sep = self.separator
        saved = sep.math
        if self.math is not None:
            sep.math = self.math
        try:
            cfg = sep.native_config(kernel_size=self.kernel_size, stride=self.stride, enc_relu=self.encoder.nonlinear)
        finally:
            sep.math = saved
        cfg.in_channels = int(self.in_channels)
        return cfg

    def native_params(self, dev):
        return self.separator.native_params(dev, enc_w=self.encoder.conv1d.weight, dec_w=self.decoder.conv_transpose1d.weight)

    def _run(self, input, want_latent):
        n_dims = input.dim()
        if n_dims == 3:
            assert input.size(1) == 1, "input.size() is expected (?, 1, ?), but given {}".format(input.size())
            if self.in_channels != 1:
                raise ValueError("a model with in_channels={} takes the 4-D input (batch, 1, n_mics, T)".format(self.in_channels))
            x = input
        elif n_dims == 4:
            # (batch, 1, n_mics, T) -> view (batch, n_mics, T) (conv_tasnet.py:138-141): the encoder consumes n_mics = in_channels
            # channels and the output gets the mic axis back (:167-168)
            assert input.size(1) == 1, "input.size() is expected (?, 1, ?, ?), but given {}".format(input.size())
            if input.size(2) != self.in_channels:
                raise ValueError("n_mics={} does not match in_channels={}".format(input.size(2), self.in_channels))
            x = input.reshape(input.size(0), input.size(2), input.size(3))
        else:
            raise ValueError("Not support {} dimension input".format(n_dims))
        training = torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())
        if training:
            from ._train import run_train, train_entry
            entry = train_entry(self)
        x = x.contiguous()
        dev = N.require_cuda(x)
        if training:
            # training: one autograd node over the whole model
            if want_latent:
                raise NotImplementedError("extract_latent under autograd is not built: call it under torch.no_grad()")
            out = run_train(self, x, entry)  # multichannel: already (B, S, C, T)
            return (out.unsqueeze(2) if n_dims == 4 and self.in_channels == 1 else out), None
        B, Cin, T = x.shape
        frames, _, _ = N.frames_of(T, self.kernel_size, self.stride)
        cfg = self.native_config()
        params, keep = self.native_params(dev)
        need = C.c_size_t(0)
        N.check(N.ctn_workspace_bytes(C.byref(cfg), B, T, C.byref(need)), "ctn_workspace_bytes")
        base, nbytes = N.aligned(N.workspace(dev, need.value))
        out = torch.empty((B, self.n_sources, Cin, T) if n_dims == 4 else (B, self.n_sources, T), dtype=torch.float32, device=dev)
        latent = torch.empty(B, self.n_sources, self.n_basis, frames, dtype=torch.float32, device=dev) if want_latent else None
        N.check(N.ctn_convtasnet_fwd(C.byref(cfg), C.byref(params), x.data_ptr(), B, T, out.data_ptr(), N.ptr(latent), base, nbytes,
                                     N.stream_ptr(dev)), "ctn_convtasnet_fwd")
        self.last_launches = N.ctn_last_launch_count()
        return out, latent
