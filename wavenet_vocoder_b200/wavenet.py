# coding: utf-8
"""``WaveNet``: the reference's class surface (wavenet.py:63-361 there) over the H100 engine.

Same constructor keywords, same ``state_dict`` keys, same helper methods, same
``incremental_forward(initial_input, c=, g=, T=, test_inputs=, tqdm=, softmax=, quantize=,
log_scale_min=)`` signature and return layout, so ``synthesis.batch_wavegen`` / ``wavegen`` /
``train.eval_model`` of the reference work unchanged with this class.  What differs is what runs:
the per-sample loop is one persistent CUDA kernel launch (csrc/wn_kernel.cuh) instead of ~600
ATen calls per sample.

Conscious divergences from the reference (SURVEY.md 7 "quirks"):
  * ``incremental_forward`` needs the module on a CUDA device; on CPU it raises (no fallback).
  * speaker ids for a batch (``g`` of shape (B,1)) are embedded per row; the reference reshapes
    them with a stale B=1 (wavenet.py:265) and fails for B>1 unless test_inputs is given.
  * sampling noise comes from a Philox generator on the device, seeded from torch's global CPU
    generator (so ``torch.manual_seed`` still makes runs reproducible); pass ``noise=`` (the
    tensors the reference would have drawn, see oracle.predraw_noise) for bit-level comparisons.
"""
from __future__ import annotations

import math
import os
from typing import Dict, Optional

import torch
from torch import nn
from torch.nn import functional as F

from . import upsample
from .engine import SynthesisEngine
from .modules import Conv1d1x1, Embedding, ResidualConv1dGLU


def receptive_field_size(total_layers, num_cycles, kernel_size, dilation=lambda x: 2 ** x):
    """(kernel_size - 1) * sum(dilations) + 1, dilations cycling ``num_cycles`` times."""
    assert total_layers % num_cycles == 0
    per = total_layers // num_cycles
    return (kernel_size - 1) * sum(dilation(i % per) for i in range(total_layers)) + 1


def _upsample_fp32(net, c):
    """The PyTorch upsample network in IEEE fp32, as the reference computes it and as the native upsampler does:
    by default cuDNN may run its convolutions in TF32 on the GPU, and on an H100 it does, which puts the head outputs
    1.2e-3 off the native path (tests/test_upsample.py::test_frames_and_sample_rate_entries_agree allows 2e-5)."""
    cudnn = torch.backends.cudnn
    with cudnn.flags(enabled=cudnn.enabled, benchmark=cudnn.benchmark, deterministic=cudnn.deterministic,
                     allow_tf32=False):
        return net(c)


def _expand_global_features(B, T, g, bct=True):
    if g is None:
        return None
    g = g.unsqueeze(-1) if g.dim() == 2 else g
    g = g.expand(B, -1, T)
    return g.contiguous() if bct else g.transpose(1, 2).contiguous()


class WaveNet(nn.Module):
    def __init__(self, out_channels=256, layers=20, stacks=2, residual_channels=512,
                 gate_channels=512, skip_out_channels=512, kernel_size=3, dropout=1 - 0.95,
                 cin_channels=-1, gin_channels=-1, n_speakers=None,
                 upsample_conditional_features=False, upsample_net="ConvInUpsampleNetwork",
                 upsample_params={"upsample_scales": [4, 4, 4, 4]}, scalar_input=False,
                 use_speaker_embedding=False, output_distribution="Logistic", cin_pad=0):
        super().__init__()
        assert layers % stacks == 0
        self.scalar_input = scalar_input
        self.out_channels = out_channels
        self.cin_channels = cin_channels
        self.gin_channels = gin_channels
        self.output_distribution = output_distribution
        self.layers, self.stacks, self.kernel_size = layers, stacks, kernel_size
        self.residual_channels, self.gate_channels = residual_channels, gate_channels
        self.skip_out_channels = skip_out_channels
        per_stack = layers // stacks
        self.first_conv = Conv1d1x1(1 if scalar_input else out_channels, residual_channels)
        self.conv_layers = nn.ModuleList([
            ResidualConv1dGLU(residual_channels, gate_channels, kernel_size=kernel_size,
                              skip_out_channels=skip_out_channels, bias=True,
                              dilation=2 ** (i % per_stack), dropout=dropout,
                              cin_channels=cin_channels, gin_channels=gin_channels)
            for i in range(layers)])
        self.last_conv_layers = nn.ModuleList([
            nn.ReLU(inplace=True), Conv1d1x1(skip_out_channels, skip_out_channels),
            nn.ReLU(inplace=True), Conv1d1x1(skip_out_channels, out_channels)])
        if gin_channels > 0 and use_speaker_embedding:
            assert n_speakers is not None
            self.embed_speakers = Embedding(n_speakers, gin_channels, padding_idx=None, std=0.1)
        else:
            self.embed_speakers = None
        if upsample_conditional_features:
            self.upsample_net = getattr(upsample, upsample_net)(**upsample_params)
        else:
            self.upsample_net = None
        self.receptive_field = receptive_field_size(layers, stacks, kernel_size)
        self._engine: Optional[SynthesisEngine] = None
        self._engine_key = None
        self._native_upsample = False

    # ------------------------------------------------------------------ small API of the reference
    def has_speaker_embedding(self):
        return self.embed_speakers is not None

    def local_conditioning_enabled(self):
        return self.cin_channels > 0

    def clear_buffer(self):
        """The engine's queues live only inside one synthesis call, so there is nothing to clear."""
        return None

    def make_generation_fast_(self):
        def strip(m):
            try:
                nn.utils.remove_weight_norm(m)
            except ValueError:
                return
        self.apply(strip)

    # ------------------------------------------------------------------ teacher-forced batch forward
    def forward(self, x, c=None, g=None, softmax=False):
        """x: (B,C,T) -> (B,out_channels,T).  Plain PyTorch (training / likelihood path)."""
        B, _, T = x.size()
        if g is not None and self.embed_speakers is not None:
            g = self.embed_speakers(g.view(B, -1)).transpose(1, 2)
            assert g.dim() == 3
        g_bct = _expand_global_features(B, T, g, bct=True)
        if c is not None and self.upsample_net is not None:
            c = self.upsample_net(c)
            assert c.size(-1) == x.size(-1)
        h = self.first_conv(x)
        skips = 0
        for layer in self.conv_layers:
            h, s = layer(h, c, g_bct)
            skips = skips + s
        h = skips * math.sqrt(1.0 / len(self.conv_layers))
        for layer in self.last_conv_layers:
            h = layer(h)
        return F.softmax(h, dim=1) if softmax else h

    # ------------------------------------------------------------------ engine management
    def _param_version(self):
        """Key of the packed-weight cache: identity and in-place version of every parameter plus a
        data-dependent fingerprint (one fused norm over all parameters), so that updates through
        ``p.data.copy_()`` / ``p.data = ...`` (EMA swaps, weight surgery), which do not bump ``_version``,
        are seen too."""
        params = list(self.parameters())
        dev = params[0].device
        norms = torch.stack(torch._foreach_norm([p.detach() for p in params])).double()
        sums = torch.stack([p.detach().reshape(-1)[0] for p in params]).double()
        finger = torch.cat([norms, sums]).cpu().numpy().tobytes()
        return (str(dev), finger) + tuple((id(p), p._version) for p in params)

    def invalidate_engine(self):
        """Forget the packed weights (they are rebuilt by the next incremental_forward)."""
        self._engine_key = None

    def load_state_dict(self, *args, **kwargs):
        self._engine_key = None
        return super().load_state_dict(*args, **kwargs)

    def _apply(self, fn, *args, **kwargs):
        self._engine_key = None
        return super()._apply(fn, *args, **kwargs)

    def __getstate__(self):
        # the engine holds ctypes handles and device buffers: never pickled / deep-copied with the module
        state = self.__dict__.copy()
        state["_engine"] = None
        state["_engine_key"] = None
        return state

    def __deepcopy__(self, memo):
        import copy
        cls = self.__class__
        new = cls.__new__(cls)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k in ("_engine", "_engine_key") else copy.deepcopy(v, memo)
        return new

    def _get_engine(self) -> SynthesisEngine:
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("WaveNet.incremental_forward runs on a CUDA device only (H100 engine, no CPU "
                               "fallback); move the model with .to('cuda')")
        key = self._param_version()
        if self._engine is None or self._engine.device != dev:
            if self._engine is not None:
                self._engine.close()
            self._engine = SynthesisEngine(
                layers=self.layers, stacks=self.stacks, residual_channels=self.residual_channels,
                gate_channels=self.gate_channels, skip_out_channels=self.skip_out_channels,
                out_channels=self.out_channels, kernel_size=self.kernel_size,
                cin_channels=self.cin_channels, gin_channels=self.gin_channels,
                scalar_input=self.scalar_input, output_distribution=self.output_distribution,
                device=dev)
            self._engine_key = None
        if self._engine_key != key:
            self._engine.load_state_dict(self.state_dict())
            # the upsample network runs on the device too when libwn covers its configuration
            self._native_upsample = self._engine.load_upsampler(self.upsample_net)
            self._engine_key = key
        return self._engine

    # ------------------------------------------------------------------ the hot path
    @torch.no_grad()
    def incremental_forward(self, initial_input=None, c=None, g=None, T=100, test_inputs=None,
                            tqdm=lambda x: x, softmax=True, quantize=True, log_scale_min=-50.0,
                            noise: Optional[Dict[str, torch.Tensor]] = None, seed=None,
                            return_params=False):
        """Autoregressive synthesis; arguments and return value as the reference's
        ``WaveNet.incremental_forward`` (wavenet.py:215-343):

        initial_input (B,C,1)|(B,1,C); c (B,C',Tc) frames (upsampled here) or (B,C',T)/(B,T,C');
        g (B,)|(B,1) speaker ids or (B,gin[,1]) features; test_inputs (B,C,T')|(B,T',C) for teacher
        forcing.  Returns (B,1,T) for scalar input, else (B,out_channels,T).
        ``log_scale_min`` is accepted and, as in the reference (mixture.py:147-148 is never
        enabled by the caller), unused.  Extensions: ``noise`` (replayed draws), ``seed``,
        ``return_params`` (also return the per-step head outputs (B,O,T)).
        """
        if self.training:
            raise RuntimeError("incremental_forward only supports eval mode")       # conv.py:19-20
        eng = self._get_engine()
        dev = eng.device
        O = self.out_channels
        B = 1
        test_scalar = test_index = test_dense = None
        if test_inputs is not None:
            ti = test_inputs.to(dev)
            if self.scalar_input:
                if ti.size(1) == 1:
                    ti = ti.transpose(1, 2)
            elif ti.size(1) == O:
                ti = ti.transpose(1, 2)
            ti = ti.contiguous().float()                                            # (B,T',C)
            B = ti.size(0)
            T = ti.size(1) if T is None else max(int(T), ti.size(1))               # wavenet.py:255-258
            if self.scalar_input:
                test_scalar = ti.reshape(B, -1)
            else:
                idx = ti.argmax(-1)
                onehot = torch.zeros_like(ti).scatter_(-1, idx.unsqueeze(-1), 1.0)
                if torch.equal(onehot, ti):
                    test_index = idx.to(torch.int32)
                else:
                    test_dense = ti
        T = int(T)
        if c is not None:
            B = c.shape[0]
        g_vec = None
        if g is not None:
            g = g.to(dev)
            if self.embed_speakers is not None:
                g_vec = self.embed_speakers(g.view(g.size(0), -1).long())[:, 0, :]   # wavenet.py:263-266
            else:
                g_vec = g.reshape(g.size(0), -1).float()
            if g_vec.size(0) == 1 and B > 1:
                g_vec = g_vec.expand(B, -1)
            B = max(B, g_vec.size(0)) if c is None and test_inputs is None else B
        c_frames = None
        if c is not None:
            c = c.to(dev).float()
            if self.upsample_net is not None and getattr(self, "_native_upsample", False) \
                    and os.environ.get("WN_TORCH_UPSAMPLE", "0") != "1":
                assert c.dim() == 3 and c.size(1) == self.cin_channels
                assert eng.upsampled_length(c.size(-1)) == T                        # wavenet.py:276
                c_frames, c = c.contiguous(), None        # conv_in + stretch/smooth run inside libwn (csrc/wn_aux.cuh)
            else:
                if self.upsample_net is not None:
                    c = _upsample_fp32(self.upsample_net, c)
                    assert c.size(-1) == T                                          # wavenet.py:276
                if c.size(-1) == T:
                    c = c.transpose(1, 2)
                c = c.contiguous()
                assert c.size(1) == T and c.size(2) == self.cin_channels
        initial = None
        initial_index = -1
        initial_rows = initial_dense = None
        if initial_input is not None and test_inputs is None:      # test_inputs override step 0 (wavenet.py:299-301)
            ii = initial_input.to(dev).float()
            if self.scalar_input:
                initial = ii.reshape(ii.size(0), -1)[:, 0].contiguous()
                if c is None and g is None:
                    B = initial.size(0)            # nothing else defines the batch (the reference assumes B=1 here)
                if initial.size(0) == 1 and B > 1:
                    initial = initial.expand(B).contiguous()
                if initial.size(0) != B:
                    raise ValueError("initial_input has %d rows but the batch is %d" % (initial.size(0), B))
            else:
                if ii.size(1) == O and ii.size(-1) != O:
                    ii = ii.transpose(1, 2)
                first = ii.reshape(ii.size(0), -1, O)[:, 0]                           # (B0, O), fed as is (wavenet.py:281-292)
                if c is None and g is None:
                    B = first.size(0)
                if first.size(0) == 1 and B > 1:
                    first = first.expand(B, -1)
                if first.size(0) != B:
                    raise ValueError("initial_input has %d rows but the batch is %d" % (first.size(0), B))
                idx = first.argmax(-1)
                onehot = torch.zeros_like(first).scatter_(-1, idx.unsqueeze(-1), 1.0)
                if torch.equal(onehot, first):
                    initial_rows = idx.to(torch.int32).contiguous()
                else:
                    initial_dense = first.contiguous()
        pinfo = eng.plan(B)
        if (self.scalar_input and B > pinfo["batch_tile"] and test_inputs is None and noise is None and not return_params
                and pinfo["engine"] == 5 and os.environ.get("WN_CONCURRENT_TILES", "1") != "0"):
            # more utterances than one batch tile, free running, device-drawn noise: two half-grid engines run two
            # tiles at the same time (engine.generate_concurrent; +23 % samples/s for 8 utterances on one H100)
            out = eng.generate_concurrent(B=B, T=T, c=c, c_frames=c_frames, g=g_vec, initial=initial, seed=seed, sync=False)
            bar = tqdm(range(T))
            eng.sync_concurrent()
            if hasattr(bar, "update"):
                bar.update(T)
            if hasattr(bar, "close"):
                bar.close()
            return out.view(B, 1, T)
        out, params = eng.generate(
            B=B, T=T, c=c, c_frames=c_frames, g=g_vec, initial=initial, initial_index=initial_index,
            initial_rows=initial_rows, initial_dense=initial_dense,
            test_scalar=test_scalar, test_index=test_index, test_dense=test_dense,
            softmax=bool(softmax), quantize=bool(quantize), noise=noise, seed=seed,
            want_params=return_params, sync=False)
        # progress-bar compatibility in O(1): the T steps are one kernel launch already in flight
        bar = tqdm(range(T))
        eng.sync()
        if hasattr(bar, "update"):
            bar.update(T)
        if hasattr(bar, "close"):
            bar.close()
        if self.scalar_input:
            y = out.view(B, 1, T)
        elif quantize:
            y = torch.zeros(B, O, T, device=dev).scatter_(1, out.long().unsqueeze(1), 1.0)
        else:
            y = out
        return (y, params) if return_params else y

    # ------------------------------------------------------------------ teacher-forced scoring on the device
    @torch.no_grad()
    def forward_native(self, x, c=None, g=None, softmax=False):
        """``forward(x, c, g, softmax)`` on the native engine (csrc/wn_dense.cuh): the same arguments and return value
        (B,out_channels,T), in eval mode and without autograd, every step computed in parallel in fp32-accurate
        (3xTF32) arithmetic.  ``c``: conditioning frames (upsampled on the device when the native upsampler covers the
        network, else by the PyTorch network in IEEE fp32) or sample-rate (B,C,T) / (B,T,C); ``g``: speaker ids or
        (B,gin[,1]) features, one vector per utterance."""
        if self.training:
            raise RuntimeError("forward_native only supports eval mode (use forward() for training)")
        if next(self.parameters()).device.type != "cuda":
            raise RuntimeError("WaveNet.forward_native runs on a CUDA device only (no CPU fallback); move the model "
                               "with .to('cuda') or use forward()")
        eng = self._get_engine()
        dev = eng.device
        O = self.out_channels
        x = x.to(dev)
        B, _, T = x.size()
        test_scalar = test_index = test_dense = None
        if self.scalar_input:
            if x.size(1) != 1:
                raise ValueError("a scalar-input model takes x of shape (B,1,T)")
            test_scalar = x[:, 0, :].float().contiguous()
        else:
            if x.size(1) != O:
                raise ValueError("a one-hot-input model takes x of shape (B,%d,T)" % O)
            xt = x.float().transpose(1, 2).contiguous()                              # (B,T,O)
            idx = xt.argmax(-1)
            if torch.equal(torch.zeros_like(xt).scatter_(-1, idx.unsqueeze(-1), 1.0), xt):
                test_index = idx.to(torch.int32)
            else:
                test_dense = xt
        g_vec = None
        if g is not None:
            g = g.to(dev)
            if self.embed_speakers is not None:
                g_vec = self.embed_speakers(g.view(B, -1).long())[:, 0, :]        # wavenet.py:187-189
            else:
                if g.dim() == 3 and g.size(-1) != 1:
                    raise ValueError("forward_native takes one global-conditioning vector per utterance")
                g_vec = g.reshape(B, -1).float()
        c_frames = None
        if c is not None:
            c = c.to(dev).float()
            if self.upsample_net is not None and self._native_upsample and \
                    os.environ.get("WN_TORCH_UPSAMPLE", "0") != "1":
                if c.dim() != 3 or c.size(1) != self.cin_channels or eng.upsampled_length(c.size(-1)) != T:
                    raise ValueError("conditioning frames %s do not upsample to T=%d" % (tuple(c.shape), T))
                c_frames, c = c.contiguous(), None
            else:
                if self.upsample_net is not None:
                    c = _upsample_fp32(self.upsample_net, c)
                if c.dim() == 3 and c.size(1) == self.cin_channels and c.size(2) == T:
                    c = c.transpose(1, 2)
                if c.dim() != 3 or c.size(0) != B or c.size(1) != T or c.size(2) != self.cin_channels:
                    raise ValueError("conditioning of shape %s does not match x (B=%d, T=%d)" % (tuple(c.shape), B, T))
                c = c.contiguous()
        return eng.forward(test_scalar=test_scalar, test_index=test_index, test_dense=test_dense, c=c,
                           c_frames=c_frames, g=g_vec, softmax=bool(softmax))

    @torch.no_grad()
    def nll(self, x, c=None, g=None, y=None, lengths=None, num_classes=65536, log_scale_min=-16.0, reduce=True):
        """Teacher-forced negative log-likelihood, as the reference's training criterion computes it
        (train.py:727-748): head outputs ``forward_native(x, c, g)[:, :, :-1]`` against targets ``y[:, 1:]``.
        ``y`` defaults to x itself: the samples for scalar input, the class ids for exactly one-hot input (otherwise
        pass ``y``, (B,T) or (B,T,1)).  ``reduce``: the mean over the mask ``sequence_mask(lengths)[:, 1:]`` (all
        samples without ``lengths``); otherwise the per-sample losses (B,T-1).  The defaults of ``num_classes`` and
        ``log_scale_min`` are the reference's hparams (quantize_channels, log_scale_min)."""
        head = self.forward_native(x, c=c, g=g, softmax=False)
        B, _, T = head.shape
        if T < 2:
            raise ValueError("nll needs T >= 2 (the head at step t scores the sample at t+1)")
        dev = head.device
        if y is None:
            if self.scalar_input:
                y = x[:, 0, :]
            else:
                xt = x.to(dev).float()
                idx = xt.argmax(1)
                if not torch.equal(torch.zeros_like(xt).scatter_(1, idx.unsqueeze(1), 1.0), xt):
                    raise ValueError("x is not exactly one-hot: pass the target classes as y")
                y = idx
        y = y.to(dev)
        if y.dim() == 3:
            y = y[:, :, 0] if y.size(-1) == 1 else y[:, 0, :]
        if tuple(y.shape) != (B, T):
            raise ValueError("y must be (B,T) = (%d,%d), got %s" % (B, T, tuple(y.shape)))
        losses = self._get_engine().nll(head[:, :, :-1].contiguous(), y[:, 1:].contiguous(), num_classes=num_classes,
                                        log_scale_min=log_scale_min)
        if not reduce:
            return losses
        if lengths is None:
            return losses.mean()
        lengths = torch.as_tensor(lengths, device=dev).long().view(-1)
        if lengths.numel() != B or int(lengths.max()) > T or int(lengths.min()) < 0:
            raise ValueError("lengths must be B values in [0, T=%d]" % T)
        mask = (torch.arange(T, device=dev).unsqueeze(0) < lengths.unsqueeze(1))[:, 1:].float()   # train.py:728-729
        return (losses * mask).sum() / mask.sum()

    # ------------------------------------------------------------------ streaming
    @torch.no_grad()
    def open_stream(self, B=1, g=None, initial_input=None, seed=None, noise=None, softmax=True, quantize=True,
                    return_params=False):
        """Synthesis in chunks: a ``WaveNetStream`` whose chunks concatenate to exactly what ``incremental_forward``
        returns for the whole utterance with the same ``g``, ``initial_input``, ``seed`` or ``noise`` (the whole
        utterance's replayed draws, sliced per chunk) and conditioning.  The state between chunks (history queues,
        fed-back sample, noise position) stays on the device.  At most one batch tile (4 utterances); no teacher
        forcing; engine 5."""
        if self.training:
            raise RuntimeError("open_stream only supports eval mode")
        return WaveNetStream(self, B=int(B), g=g, initial_input=initial_input, seed=seed, noise=noise,
                             softmax=softmax, quantize=quantize, return_params=return_params)


class WaveNetStream:
    """Chunks of one utterance (or a batch tile of them) from ``WaveNet.open_stream``.

    ``generate(T, c=)`` takes sample-rate conditioning; ``push_frames(frames)`` takes conditioning frames as they
    arrive and returns the samples whose frames are all known (possibly none); ``finish()`` returns the rest, up to
    the upsampled length of all frames pushed.  Outputs are laid out as ``incremental_forward``'s."""

    def __init__(self, model, *, B, g, initial_input, seed, noise, softmax, quantize, return_params):
        self._m = model
        self._eng = eng = model._get_engine()
        dev = eng.device
        O = model.out_channels
        g_vec = None
        if g is not None:
            g = g.to(dev)
            if model.embed_speakers is not None:
                g_vec = model.embed_speakers(g.view(g.size(0), -1).long())[:, 0, :]   # wavenet.py:263-266
            else:
                g_vec = g.reshape(g.size(0), -1).float()
            if g_vec.size(0) == 1 and B > 1:
                g_vec = g_vec.expand(B, -1)
        initial = initial_rows = initial_dense = None
        if initial_input is not None:
            ii = initial_input.to(dev).float()
            if model.scalar_input:
                initial = ii.reshape(ii.size(0), -1)[:, 0]
                initial = initial.expand(B) if initial.size(0) == 1 else initial
            else:
                if ii.size(1) == O and ii.size(-1) != O:
                    ii = ii.transpose(1, 2)
                first = ii.reshape(ii.size(0), -1, O)[:, 0]
                first = first.expand(B, -1) if first.size(0) == 1 else first
                idx = first.argmax(-1)
                if torch.equal(torch.zeros_like(first).scatter_(-1, idx.unsqueeze(-1), 1.0), first):
                    initial_rows = idx.to(torch.int32)
                else:
                    initial_dense = first
        self._noise = None if noise is None else {k: v.to(dev) for k, v in noise.items()}
        self._s = eng.open_stream(B=B, g=g_vec, initial=initial, initial_rows=initial_rows, initial_dense=initial_dense,
                                  softmax=bool(softmax), quantize=bool(quantize), replay=noise is not None, seed=seed)
        self.B, self._quantize, self._return_params = B, bool(quantize), bool(return_params)
        self._frames = None          # every frame pushed so far, (B,C,n) on the device
        self._finished = False

    @property
    def t(self) -> int:
        """Samples generated so far."""
        return self._s.t

    def close(self):
        self._s.close()

    def _chunk(self, T, **kw):
        if self._finished:
            raise RuntimeError("the stream was finished")
        if self._m._get_engine() is not self._eng:      # reloads changed weights: the library then refuses the chunk
            raise RuntimeError("the model moved to another device since the stream was opened")
        t = self.t
        noise = None if self._noise is None else {k: v[t:t + T] for k, v in self._noise.items()}
        out, params = self._s.generate(T, noise=noise, want_params=self._return_params, **kw)
        B, O = self.B, self._m.out_channels
        if self._m.scalar_input:
            y = out.view(B, 1, T)
        elif self._quantize:
            y = torch.zeros(B, O, T, device=out.device).scatter_(1, out.long().unsqueeze(1), 1.0)
        else:
            y = out
        return (y, params) if self._return_params else y

    def _empty(self):
        dev = self._eng.device
        C = 1 if self._m.scalar_input else self._m.out_channels
        y = torch.zeros(self.B, C, 0, device=dev)
        return (y, torch.zeros(self.B, self._m.out_channels, 0, device=dev)) if self._return_params else y

    @torch.no_grad()
    def generate(self, T, c=None):
        """The next T samples; ``c``: their sample-rate conditioning, (B,C,T) or (B,T,C)."""
        T = int(T)
        if c is not None:
            c = c.to(self._eng.device).float()
            if c.size(-1) == T and c.size(1) == self._m.cin_channels:
                c = c.transpose(1, 2)
            c = c.contiguous()
        return self._chunk(T, c=c)

    @torch.no_grad()
    def push_frames(self, frames):
        """Append conditioning frames (B,C,n) and return the samples they complete (possibly none)."""
        frames = frames.to(self._eng.device).float()
        if self._m.upsample_net is None:
            return self.generate(frames.size(-1), c=frames)       # frames are at the sample rate already
        if not self._m._native_upsample:
            raise RuntimeError("push_frames needs an upsample network the native upsampler covers (engine.upsampler_struct)")
        self._frames = frames if self._frames is None else torch.cat([self._frames, frames], dim=-1)
        return self._frames_chunk(final=False)

    @torch.no_grad()
    def finish(self):
        """The samples left once no further frame follows, up to the upsampled length of all frames pushed."""
        if self._m.upsample_net is None or self._frames is None:
            self._finished = True
            return self._empty()
        out = self._frames_chunk(final=True)
        self._finished = True
        return out

    def _frames_chunk(self, final):
        n = self._frames.size(-1)
        t = self.t
        _, _, ready = self._eng.upsample_cone(n, final)
        if ready <= t:
            return self._empty()
        f_lo, f_hi, _ = self._eng.upsample_cone(n, final, t, ready)
        return self._chunk(ready - t, c_frames=self._frames[:, :, f_lo:f_hi], frame_offset=f_lo, frames_total=n,
                           final=final)
