# coding: utf-8
"""Thin host wrapper around one libwn handle: weights in, one synthesis call out.

PyTorch is used for device memory and streams only; all arithmetic of the path happens inside
libwn.so (csrc/wn_kernel.cuh).  Mirrors the data the reference loop consumes
(wavenet.py:215-343): upsampled local conditioning (B,T,C), embedded global conditioning (B,gin),
optional teacher-forcing inputs, and returns the generated samples.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Dict, Optional

import torch

from . import _native as N


def fold_weight_norm(sd: Dict[str, torch.Tensor], prefix: str) -> torch.Tensor:
    """w = g * v / ||v|| over all dims but 0 (the reference wraps every conv in weight_norm,
    modules.py:13-18); accepts the stripped form left by make_generation_fast_ (wavenet.py:355-361)."""
    if prefix + ".weight" in sd:
        return sd[prefix + ".weight"].detach().float().cpu()
    g = sd[prefix + ".weight_g"].detach().float().cpu()
    v = sd[prefix + ".weight_v"].detach().float().cpu()
    return torch._weight_norm(v, g, 0)


def linearize(w: torch.Tensor) -> torch.Tensor:
    """(out, in, kw) -> (out, kw*in), tap-major: the order conv.py:51-62 feeds to F.linear."""
    return w.transpose(1, 2).contiguous().view(w.size(0), -1).contiguous()


def weights_struct(sd: Dict[str, torch.Tensor], layers: int, cin: int, gin: int):
    """state_dict (weight-normed or stripped) -> (wn_weights of HOST pointers, keep-alive list)."""
    keep = []

    def ptr(t: Optional[torch.Tensor]):
        if t is None:
            return None
        t = t.detach().float().cpu().contiguous()
        keep.append(t)
        return C.cast(t.data_ptr(), C.POINTER(C.c_float))

    def conv(prefix):
        return linearize(fold_weight_norm(sd, prefix))

    def bias(prefix):
        return sd.get(prefix + ".bias")

    lw = (N.wn_layer_weights * layers)()
    for i in range(layers):
        p = "conv_layers.%d." % i
        lw[i].conv_w = ptr(conv(p + "conv"))
        lw[i].conv_b = ptr(bias(p + "conv"))
        lw[i].cond_w = ptr(conv(p + "conv1x1c")) if cin > 0 else None
        lw[i].gcond_w = ptr(conv(p + "conv1x1g")) if gin > 0 else None
        lw[i].out_w = ptr(conv(p + "conv1x1_out"))
        lw[i].out_b = ptr(bias(p + "conv1x1_out"))
        lw[i].skip_w = ptr(conv(p + "conv1x1_skip"))
        lw[i].skip_b = ptr(bias(p + "conv1x1_skip"))
    w = N.wn_weights()
    w.first_w = ptr(conv("first_conv"))
    w.first_b = ptr(bias("first_conv"))
    w.last_a_w = ptr(conv("last_conv_layers.1"))
    w.last_a_b = ptr(bias("last_conv_layers.1"))
    w.last_b_w = ptr(conv("last_conv_layers.3"))
    w.last_b_b = ptr(bias("last_conv_layers.3"))
    w.layers = lw
    keep.append(lw)
    return w, keep


def make_config(*, layers, stacks, residual_channels, gate_channels, skip_out_channels, out_channels,
                kernel_size, cin_channels, gin_channels, scalar_input, output_distribution,
                device_index=0, num_ctas=0, exchange_copies=0, ring_slots=0, poll_warps=0, engine=0):
    """wn_config from the reference's constructor keywords (wavenet.py:98-111).  num_ctas, exchange_copies,
    ring_slots and poll_warps are the planner's fields of include/wn.h (0 = the planner chooses); engine is the kernel
    organisation (0 = WN_ENGINE, else 5; 5 or 7 = that one)."""
    if scalar_input:
        if output_distribution == "Logistic":
            head = N.WN_HEAD_MOL
        elif output_distribution == "Normal":
            head = N.WN_HEAD_GAUSS
        else:
            raise AssertionError(output_distribution)      # wavenet.py:329-330
    else:
        head = N.WN_HEAD_SOFTMAX
    cfg = N.wn_config()
    cfg.abi_version = N.WN_ABI_VERSION
    cfg.layers, cfg.stacks = int(layers), int(stacks)
    cfg.residual_channels, cfg.gate_channels = int(residual_channels), int(gate_channels)
    cfg.skip_channels, cfg.out_channels = int(skip_out_channels), int(out_channels)
    cfg.kernel_size = int(kernel_size)
    cfg.cin_channels, cfg.gin_channels = max(int(cin_channels), 0), max(int(gin_channels), 0)
    cfg.input_kind = N.WN_INPUT_SCALAR if scalar_input else N.WN_INPUT_ONEHOT
    cfg.head_kind = head
    cfg.device = int(device_index)
    cfg.num_ctas = int(num_ctas)
    cfg.exchange_copies, cfg.ring_slots, cfg.poll_warps = int(exchange_copies), int(ring_slots), int(poll_warps)
    cfg.engine = int(engine)
    return cfg


def upsampler_struct(net, cin):
    """The wn_upsampler of a PyTorch upsample network (upsample.py), or None for a variant the native path does not
    cover.  Returns {"u": wn_upsampler, "total", "frames_lost", "indent"}; the struct's arrays are kept in the dict."""
    from . import upsample as U
    if net is None or cin <= 0:
        return None
    conv_in = None
    up = net
    if isinstance(net, U.ConvInUpsampleNetwork):
        conv_in, up = net.conv_in, net.upsample
    if not isinstance(up, U.UpsampleNetwork):
        return None
    scales, filters = [], []
    layers = list(up.up_layers)
    if len(layers) % 2 != 0:
        return None                                    # an activation follows every conv
    for st, conv in zip(layers[0::2], layers[1::2]):
        if not isinstance(st, U.Stretch2d) or st.mode != "nearest" or st.y_scale != 1:
            return None
        sd = {k: v for k, v in conv.state_dict().items()}
        if "weight" in sd:
            w = sd["weight"].detach().float().cpu()
        else:
            w = torch._weight_norm(sd["weight_v"].detach().float().cpu(), sd["weight_g"].detach().float().cpu(), 0)
        s = int(st.x_scale)
        if w.shape != (1, 1, 1, 2 * s + 1) or s < 2:
            return None
        scales.append(s)
        filters.append(w.reshape(-1))
    if not scales or len(scales) > 8:
        return None
    u = N.wn_upsampler()
    u.channels = cin
    u.n_scales = len(scales)
    sc = (C.c_int32 * len(scales))(*scales)
    fl = torch.cat(filters).contiguous()
    u.scales = sc
    u.filters = C.cast(fl.data_ptr(), C.POINTER(C.c_float))
    cw = None
    if conv_in is not None:
        cw = conv_in.weight.detach().float().cpu().contiguous()
        if cw.shape[0] != cin or cw.shape[1] != cin or conv_in.bias is not None:
            return None
        u.conv_in_w = C.cast(cw.data_ptr(), C.POINTER(C.c_float))
        u.conv_in_ks = int(cw.shape[2])
    u.indent = int(up.indent)
    total = 1
    for s in scales:
        total *= s
    return dict(u=u, keep=(sc, fl, cw), total=total, frames_lost=int(cw.shape[2]) - 1 if cw is not None else 0,
                indent=int(up.indent))


def upsample_cone(u, n_frames, final, t_lo=0, t_hi=0):
    """wn_upsample_cone (no device needed): (f_lo, f_hi, n_ready)."""
    f_lo, f_hi, n_ready = C.c_int64(), C.c_int64(), C.c_int64()
    N.check(N.lib().wn_upsample_cone(C.byref(u), int(n_frames), int(bool(final)), int(t_lo), int(t_hi), C.byref(f_lo),
                                     C.byref(f_hi), C.byref(n_ready)))
    return f_lo.value, f_hi.value, n_ready.value


def nll(head: torch.Tensor, head_kind: int, target: torch.Tensor, num_classes: int = 65536,
        log_scale_min: float = -16.0) -> torch.Tensor:
    """wn_nll: per-sample negative log-likelihood (B,T) of ``target`` under head outputs ``head`` (B,O,T) on a CUDA
    device -- the reference's discretized_mix_logistic_loss / mix_gaussian_loss / cross-entropy with reduce=False.
    ``target``: (B,T) samples in [-1,1] for a MoL or Gaussian head, (B,T) class ids for a softmax head."""
    if head.device.type != "cuda" or head.dim() != 3:
        raise ValueError("head must be a (B,O,T) CUDA tensor")
    B, O, T = head.shape
    y = head.float().contiguous()
    if tuple(target.shape) != (B, T):
        raise ValueError("target must be (B,T) = (%d,%d), got %s" % (B, T, tuple(target.shape)))
    yt = ct = None
    if head_kind == N.WN_HEAD_SOFTMAX:
        ct = target.to(device=head.device, dtype=torch.int32).contiguous()
    else:
        yt = target.to(device=head.device, dtype=torch.float32).contiguous()
    out = torch.empty(B, T, device=head.device, dtype=torch.float32)
    stream = torch.cuda.current_stream(head.device)
    N.check(N.lib().wn_nll(y.data_ptr(), int(head_kind), B, O, T, None if yt is None else yt.data_ptr(),
                           None if ct is None else ct.data_ptr(), int(num_classes), float(log_scale_min),
                           out.data_ptr(), stream.cuda_stream))
    return out


class SynthesisStream:
    """One utterance (or one batch tile of them) made chunk by chunk; the state between chunks stays on the device
    (wn_stream_* of include/wn.h).  Chunks are bit-identical to the same samples of one ``generate`` call on the same
    handle.  ``engine``: 0 or 5 = an engine-5 stream (1..4 utterances), 7 = an engine-7 stream (1..8 utterances) on a
    handle that runs engine 7."""

    def __init__(self, eng, *, B, g=None, initial=None, initial_index=-1, initial_rows=None, initial_dense=None,
                 softmax=True, quantize=True, replay=False, seed=None, philox_row0=0, engine=0):
        self.eng, self.B, self.quantize = eng, int(B), bool(quantize)
        dev = eng.device
        a = N.wn_stream_open_args()
        a.B = self.B
        a.engine = int(engine)
        hold = []

        def dptr(t, dtype=torch.float32, shape=None):
            if t is None:
                return None
            t = t.to(device=dev, dtype=dtype).contiguous()
            if shape is not None and tuple(t.shape) != tuple(shape):
                raise ValueError("expected shape %s, got %s" % (tuple(shape), tuple(t.shape)))
            hold.append(t)
            return t.data_ptr()

        a.g = dptr(g, shape=(B, eng.gin) if g is not None else None)
        a.initial = dptr(initial, shape=(B,) if initial is not None else None)
        a.initial_index = int(initial_index)
        a.initial_rows = dptr(initial_rows, torch.int32, shape=(B,) if initial_rows is not None else None)
        a.initial_dense = dptr(initial_dense, shape=(B, eng.out_channels) if initial_dense is not None else None)
        a.flags = (N.WN_FLAG_SOFTMAX if softmax else 0) | (N.WN_FLAG_QUANTIZE if quantize else 0)
        if replay:
            a.noise_kind = N.WN_NOISE_REPLAY
        else:
            a.noise_kind = N.WN_NOISE_PHILOX
            if seed is None:
                seed = int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())
            a.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        a.philox_row0 = int(philox_row0)
        a.stream = torch.cuda.current_stream(dev).cuda_stream
        self._s = C.c_void_p()
        N.check(N.lib().wn_stream_open(eng._h, C.byref(a), C.byref(self._s)))   # returns after the set-up ran
        eng._streams.add(self)

    @property
    def t(self) -> int:
        """Samples generated so far (the absolute step of the next one)."""
        self._check_open()
        return int(N.lib().wn_stream_position(self._s))

    def _check_open(self):
        if not self._s.value:
            raise RuntimeError("the stream is closed")

    def generate(self, T, *, c=None, c_frames=None, frame_offset=0, frames_total=0, final=False, noise=None,
                 want_params=False, sync=True):
        """The next T samples.  c: (B,T,C) sample-rate conditioning of these samples; or c_frames (B,C,n), utterance
        frames [frame_offset, frame_offset+n) of the frames_total received so far (``final``: all of them).
        noise: these T steps' replayed draws, (T,B,.).  Returns (out, params) as SynthesisEngine.generate."""
        self._check_open()
        eng, B, dev, O = self.eng, self.B, self.eng.device, self.eng.out_channels
        a = N.wn_generate_args()
        a.B, a.T = B, int(T)
        hold = []

        def dptr(t, shape=None):
            if t is None:
                return None
            t = t.to(device=dev, dtype=torch.float32).contiguous()
            if shape is not None and tuple(t.shape) != tuple(shape):
                raise ValueError("expected shape %s, got %s" % (tuple(shape), tuple(t.shape)))
            hold.append(t)
            return t.data_ptr()

        a.c = dptr(c, shape=(B, T, eng.cin) if c is not None else None)
        where = None
        if c_frames is not None:
            a.c_frames = dptr(c_frames, shape=(B, eng.cin, c_frames.size(-1)))
            a.n_frames = int(c_frames.size(-1))
        if c_frames is not None or final:
            where = N.wn_stream_chunk()
            where.frame_offset, where.frames_total, where.final = int(frame_offset), int(frames_total), int(bool(final))
        if noise is not None:
            a.noise_u1 = dptr(noise.get("u1"), shape=(T, B, eng.K) if "u1" in noise else None)
            a.noise_u2 = dptr(noise.get("u2"), shape=(T, B) if "u2" in noise else None)
            a.noise_z = dptr(noise.get("z"), shape=(T, B) if "z" in noise else None)
            a.noise_e = dptr(noise.get("e"), shape=(T, B, O) if "e" in noise else None)
        if eng.scalar_input:
            out = torch.empty(B, T, device=dev, dtype=torch.float32)
            a.out_scalar = out.data_ptr()
        elif self.quantize:
            out = torch.empty(B, T, device=dev, dtype=torch.int32)
            a.out_index = out.data_ptr()
        else:
            out = torch.empty(B, O, T, device=dev, dtype=torch.float32)
            a.out_dense = out.data_ptr()
        params = None
        if want_params:
            params = torch.empty(B, O, T, device=dev, dtype=torch.float32)
            a.params_out = params.data_ptr()
        a.stream = torch.cuda.current_stream(dev).cuda_stream
        N.check(N.lib().wn_stream_generate(self._s, C.byref(a), None if where is None else C.byref(where)))
        eng._keep = hold
        if sync:
            eng.sync()
        return out, params

    def close(self):
        if getattr(self, "_s", None) is not None and self._s.value:
            N.lib().wn_stream_close(self._s)
            self._s = C.c_void_p()
            self.eng._streams.discard(self)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SynthesisEngine:
    """One model shape on one GPU."""

    def __init__(self, *, layers, stacks, residual_channels, gate_channels, skip_out_channels,
                 out_channels, kernel_size, cin_channels, gin_channels, scalar_input,
                 output_distribution, device: torch.device, num_ctas=0, exchange_copies=0, ring_slots=0,
                 poll_warps=0, engine=0):
        if device.type != "cuda":
            raise RuntimeError("wavenet_vocoder_b200 runs the synthesis path on a CUDA device only "
                               "(there is no CPU fallback); got device %s" % device)
        self.device = device
        self.scalar_input = bool(scalar_input)
        self.out_channels = int(out_channels)
        self.cin = max(int(cin_channels), 0)
        self.gin = max(int(gin_channels), 0)
        cfg = make_config(layers=layers, stacks=stacks, residual_channels=residual_channels,
                          gate_channels=gate_channels, skip_out_channels=skip_out_channels,
                          out_channels=out_channels, kernel_size=kernel_size, cin_channels=cin_channels,
                          gin_channels=gin_channels, scalar_input=scalar_input,
                          output_distribution=output_distribution,
                          device_index=device.index if device.index is not None else torch.cuda.current_device(),
                          num_ctas=num_ctas, exchange_copies=exchange_copies, ring_slots=ring_slots,
                          poll_warps=poll_warps, engine=engine)
        self.head = head = cfg.head_kind
        self.K = 0 if head == N.WN_HEAD_SOFTMAX else (1 if out_channels == 2 else out_channels // 3)
        self.cfg = cfg
        self._h = C.c_void_p()
        N.check(N.lib().wn_create(C.byref(cfg), C.byref(self._h)))
        self._keep = None
        self._ctor = dict(layers=layers, stacks=stacks, residual_channels=residual_channels, gate_channels=gate_channels,
                          skip_out_channels=skip_out_channels, out_channels=out_channels, kernel_size=kernel_size,
                          cin_channels=cin_channels, gin_channels=gin_channels, scalar_input=scalar_input,
                          output_distribution=output_distribution, device=device,
                          exchange_copies=exchange_copies, ring_slots=ring_slots, poll_warps=poll_warps, engine=engine)
        self._sd = None
        self._halves = None           # two half-grid engines for concurrent batch tiles (see generate_concurrent)
        self._sib7 = None             # an engine-7 engine of the same model for engine-7 streams (see engine7)
        self._is_child = num_ctas > 0
        self._ups = None
        self._streams = weakref.WeakSet()   # open SynthesisStreams: closed before the handle they run on

    def close(self):
        for s in list(getattr(self, "_streams", None) or []):
            s.close()
        for ch in (getattr(self, "_halves", None) or []):
            ch["eng"].close()
        self._halves = None
        if getattr(self, "_sib7", None) is not None:
            self._sib7.close()
        self._sib7 = None
        if getattr(self, "_h", None) is not None and self._h.value:
            N.lib().wn_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        """Fold weight norm, linearise the dilated convs, hand the host arrays to libwn."""
        w, keep = weights_struct(sd, self.cfg.layers, self.cin, self.gin)
        N.check(N.lib().wn_load_weights(self._h, C.byref(w)))
        del keep
        if not self._is_child:
            self._sd = {k: v.detach().cpu() for k, v in sd.items() if not k.startswith("upsample_net.")}
            for ch in (self._halves or []):
                ch["eng"].close()
            self._halves = None
            if self._sib7 is not None:
                # reloaded, not closed: its open streams then refuse their next chunk (the weights changed)
                self._sib7.load_state_dict(sd)

    def load_upsampler(self, net) -> bool:
        """Hand the local-conditioning upsampler (upsample.py:29-85 there) to libwn so that ``generate`` can take
        raw conditioning frames.  Returns False (and unloads) for variants the native path does not cover
        (freq_axis_kernel_size != 1, an activation, a non-nearest mode, a scale < 2): the caller then keeps
        them on the PyTorch side and passes sample-rate ``c``."""
        self._ups_net = net
        for ch in (getattr(self, "_halves", None) or []):
            ch["eng"].load_upsampler(net)
        if getattr(self, "_sib7", None) is not None:
            self._sib7.load_upsampler(net)
        self.ups_frames_lost = 0
        self.ups_total = 1
        self._ups = None
        N.check(N.lib().wn_load_upsampler(self._h, None))
        d = upsampler_struct(net, self.cin)
        if d is None:
            return False
        N.check(N.lib().wn_load_upsampler(self._h, C.byref(d["u"])))
        self._ups = d
        self.ups_total = d["total"]
        self.ups_frames_lost = d["frames_lost"]
        self.ups_indent = d["indent"]
        return True

    def upsample_cone(self, n_frames: int, final: bool, t_lo: int = 0, t_hi: int = 0):
        """(f_lo, f_hi, n_ready): the frames [f_lo, f_hi) samples [t_lo, t_hi) need, and how many samples from the
        start are known from ``n_frames`` frames (``final``: all of them); libwn's wn_upsample_cone."""
        if self._ups is None:
            raise RuntimeError("no native upsampler is loaded")
        return upsample_cone(self._ups["u"], n_frames, final, t_lo, t_hi)

    def upsample(self, c_frames: torch.Tensor, T: int) -> torch.Tensor:
        """(B,C,frames) -> (B,T,C): only the upsampler of libwn (tests / tools)."""
        B = c_frames.size(0)
        cf = c_frames.to(device=self.device, dtype=torch.float32).contiguous()
        out = torch.empty(B, T, self.cin, device=self.device, dtype=torch.float32)
        N.check(N.lib().wn_upsample(self._h, cf.data_ptr(), B, int(cf.size(-1)), int(T), out.data_ptr(),
                                    torch.cuda.current_stream(self.device).cuda_stream))
        torch.cuda.current_stream(self.device).synchronize()
        return out

    def upsampled_length(self, n_frames: int) -> int:
        return (n_frames - self.ups_frames_lost) * self.ups_total - 2 * self.ups_indent

    def plan(self, batch=1) -> dict:
        info = N.wn_plan_info()
        N.check(N.lib().wn_get_plan(self._h, int(batch), C.byref(info)))
        return info.as_dict()

    # ------------------------------------------------------------------ one synthesis call
    def generate(self, *, B: int, T: int, c: Optional[torch.Tensor] = None,
                 c_frames: Optional[torch.Tensor] = None, g: Optional[torch.Tensor] = None, initial: Optional[torch.Tensor] = None,
                 initial_index: int = -1, initial_rows: Optional[torch.Tensor] = None,
                 initial_dense: Optional[torch.Tensor] = None, test_scalar: Optional[torch.Tensor] = None,
                 test_index: Optional[torch.Tensor] = None,
                 test_dense: Optional[torch.Tensor] = None, softmax=True, quantize=True,
                 noise: Optional[Dict[str, torch.Tensor]] = None, seed: Optional[int] = None,
                 want_params=False, sync=True, philox_row0: int = 0):
        """All tensors on self.device, fp32 (indices int32), contiguous in the layouts of
        include/wn.h.  Returns (out, params) where out is (B,T) float, (B,T) int32 or (B,O,T)."""
        dev = self.device
        O = self.out_channels
        a = N.wn_generate_args()
        a.B, a.T = int(B), int(T)
        a.philox_row0 = int(philox_row0)
        hold = []

        def dptr(t, dtype=torch.float32, shape=None):
            if t is None:
                return None
            t = t.to(device=dev, dtype=dtype).contiguous()
            if shape is not None and tuple(t.shape) != tuple(shape):
                raise ValueError("expected shape %s, got %s" % (tuple(shape), tuple(t.shape)))
            hold.append(t)
            return t.data_ptr()

        a.c = dptr(c, shape=(B, T, self.cin) if c is not None else None)
        if c_frames is not None:
            a.c_frames = dptr(c_frames, shape=(B, self.cin, c_frames.size(-1)))
            a.n_frames = int(c_frames.size(-1))
        a.g = dptr(g, shape=(B, self.gin) if g is not None else None)
        a.initial = dptr(initial, shape=(B,) if initial is not None else None)
        a.initial_index = int(initial_index)
        a.initial_rows = dptr(initial_rows, torch.int32, shape=(B,) if initial_rows is not None else None)
        a.initial_dense = dptr(initial_dense, shape=(B, O) if initial_dense is not None else None)
        T_test = 0
        if test_scalar is not None:
            T_test = test_scalar.size(1)
            a.test_scalar = dptr(test_scalar, shape=(B, T_test))
        if test_index is not None:
            T_test = test_index.size(1)
            a.test_index = dptr(test_index, torch.int32, shape=(B, T_test))
        if test_dense is not None:
            T_test = test_dense.size(1)
            a.test_dense = dptr(test_dense, shape=(B, T_test, O))
        a.T_test = int(T_test)
        a.flags = (N.WN_FLAG_SOFTMAX if softmax else 0) | (N.WN_FLAG_QUANTIZE if quantize else 0)
        if noise is not None:
            a.noise_kind = N.WN_NOISE_REPLAY
            a.noise_u1 = dptr(noise.get("u1"), shape=(T, B, self.K) if "u1" in noise else None)
            a.noise_u2 = dptr(noise.get("u2"), shape=(T, B) if "u2" in noise else None)
            a.noise_z = dptr(noise.get("z"), shape=(T, B) if "z" in noise else None)
            a.noise_e = dptr(noise.get("e"), shape=(T, B, O) if "e" in noise else None)
        else:
            a.noise_kind = N.WN_NOISE_PHILOX
            if seed is None:
                # deterministic under torch.manual_seed, like the reference's use of the global RNG
                seed = int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())
            a.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        out = None
        if self.scalar_input:
            out = torch.empty(B, T, device=dev, dtype=torch.float32)
            a.out_scalar = out.data_ptr()
        elif quantize:
            out = torch.empty(B, T, device=dev, dtype=torch.int32)
            a.out_index = out.data_ptr()
        else:
            out = torch.empty(B, O, T, device=dev, dtype=torch.float32)
            a.out_dense = out.data_ptr()
        params = None
        if want_params:
            params = torch.empty(B, O, T, device=dev, dtype=torch.float32)
            a.params_out = params.data_ptr()
        a.stream = torch.cuda.current_stream(dev).cuda_stream
        N.check(N.lib().wn_generate(self._h, C.byref(a)))
        self._keep = hold          # inputs must outlive the asynchronous launch
        if sync:
            self.sync()
        return out, params

    # ------------------------------------------------------------------ teacher-forced scoring
    def forward(self, *, test_scalar: Optional[torch.Tensor] = None, test_index: Optional[torch.Tensor] = None,
                test_dense: Optional[torch.Tensor] = None, c: Optional[torch.Tensor] = None,
                c_frames: Optional[torch.Tensor] = None, g: Optional[torch.Tensor] = None, softmax=False, sync=True):
        """Teacher-forced batch forward (wn_forward): the head outputs (B,O,T) of every step, computed in parallel over
        time.  The input is exactly one of test_scalar (B,T), test_index (B,T) class ids or test_dense (B,T,O); c, c_frames
        and g as in ``generate``; ``softmax`` applies a softmax over O."""
        given = [t for t in (test_scalar, test_index, test_dense) if t is not None]
        if len(given) != 1:
            raise ValueError("give exactly one of test_scalar, test_index, test_dense")
        dev, O = self.device, self.out_channels
        B, T = int(given[0].size(0)), int(given[0].size(1))
        a = N.wn_generate_args()
        a.B, a.T, a.T_test = B, T, T
        hold = []

        def dptr(t, dtype=torch.float32, shape=None):
            if t is None:
                return None
            t = t.to(device=dev, dtype=dtype).contiguous()
            if shape is not None and tuple(t.shape) != tuple(shape):
                raise ValueError("expected shape %s, got %s" % (tuple(shape), tuple(t.shape)))
            hold.append(t)
            return t.data_ptr()

        a.test_scalar = dptr(test_scalar, shape=(B, T))
        a.test_index = dptr(test_index, torch.int32, shape=(B, T))
        a.test_dense = dptr(test_dense, shape=(B, T, O))
        a.c = dptr(c, shape=(B, T, self.cin) if c is not None else None)
        if c_frames is not None:
            a.c_frames = dptr(c_frames, shape=(B, self.cin, c_frames.size(-1)))
            a.n_frames = int(c_frames.size(-1))
        a.g = dptr(g, shape=(B, self.gin) if g is not None else None)
        a.initial_index = -1
        a.flags = N.WN_FLAG_SOFTMAX if softmax else 0
        params = torch.empty(B, O, T, device=dev, dtype=torch.float32)
        a.params_out = params.data_ptr()
        a.stream = torch.cuda.current_stream(dev).cuda_stream
        N.check(N.lib().wn_forward(self._h, C.byref(a)))
        self._keep = hold
        if sync:
            self.sync()
        return params

    def nll(self, head: torch.Tensor, target: torch.Tensor, num_classes: int = 65536,
            log_scale_min: float = -16.0) -> torch.Tensor:
        """Per-sample negative log-likelihood (B,T) of ``target`` under head outputs (B,O,T) of this model's output
        head (wn_nll); see ``nll``."""
        return nll(head, self.head, target, num_classes=num_classes, log_scale_min=log_scale_min)

    # ------------------------------------------------------------------ streaming
    def open_stream(self, **kw) -> SynthesisStream:
        """A stream of chunks on this handle (keywords of SynthesisStream); one batch tile.  ``engine=7`` opens an
        engine-7 stream of up to 8 utterances, which needs a handle created with ``engine=7``."""
        return SynthesisStream(self, **kw)

    def engine7(self) -> "SynthesisEngine":
        """This engine if it runs engine 7, else an engine-7 engine of the same model on the same device, made on
        first use with this engine's weights and upsampler, reloaded with them and closed with this engine."""
        if self.plan(1)["engine"] == 7:
            return self
        if self._sib7 is None:
            if self._sd is None:
                raise RuntimeError("load_state_dict first")
            e = SynthesisEngine(**dict(self._ctor, engine=7))
            e._is_child = True            # its weights are this engine's: nothing to keep twice
            e.load_state_dict(self._sd)
            if getattr(self, "_ups_net", None) is not None:
                e.load_upsampler(self._ups_net)
            self._sib7 = e
        return self._sib7

    # ------------------------------------------------------------------ two batch tiles at a time
    def generate_concurrent(self, *, B: int, T: int, c: Optional[torch.Tensor] = None,
                            c_frames: Optional[torch.Tensor] = None, g: Optional[torch.Tensor] = None,
                            initial: Optional[torch.Tensor] = None, seed: Optional[int] = None, sync=True):
        """Free-running synthesis of B > one tile of utterances with device-drawn noise: two HALF-GRID engines (64
        blocks each) run two batch tiles at the same time on two streams, instead of one full-grid launch per tile one
        after the other (BASELINE config 4's per-GPU share of 8 utterances is two tiles of 4).  A step of the sample
        loop is latency-bound, not SM-bound, so two half-grid chains overlap (+23 % samples/s for 8 utterances on an H100 SXM).  Utterances are
        independent and row b draws the Philox noise of row b of a single call with the same seed (``philox_row0``), so
        the result is that of ``generate(B=B, seed=seed)`` up to fp32 summation order.  Returns (B,T) samples."""
        if not self.scalar_input:
            raise ValueError("generate_concurrent supports scalar-input models")
        plan = self.plan(1)
        half = max(1, plan["num_ctas"] // 2)
        tile = 4
        if self._halves is None:
            if self._sd is None:
                raise RuntimeError("load_state_dict first")
            self._halves = []
            for _ in range(2):
                e = SynthesisEngine(num_ctas=half, **self._ctor)
                e.load_state_dict(self._sd)
                if getattr(self, "_ups_net", None) is not None:
                    e.load_upsampler(self._ups_net)
                self._halves.append(dict(eng=e, stream=torch.cuda.Stream(device=self.device)))
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,), dtype=torch.int64).item())
        dev = self.device
        out = torch.empty(B, T, device=dev, dtype=torch.float32)
        cur = torch.cuda.current_stream(dev)
        ready = torch.cuda.Event()
        ready.record(cur)
        hold = [c, c_frames, g, initial, out]
        for k, b0 in enumerate(range(0, B, tile)):
            ch = self._halves[k % 2]
            Bc = min(tile, B - b0)
            ch["stream"].wait_event(ready)
            with torch.cuda.stream(ch["stream"]):
                o, _ = ch["eng"].generate(B=Bc, T=T, c=None if c is None else c[b0:b0 + Bc],
                                          c_frames=None if c_frames is None else c_frames[b0:b0 + Bc].contiguous(),
                                          g=None if g is None else g[b0:b0 + Bc].contiguous(),
                                          initial=None if initial is None else initial[b0:b0 + Bc].contiguous(),
                                          seed=seed, philox_row0=b0, sync=False)
                out[b0:b0 + Bc].copy_(o, non_blocking=True)
                hold.append(o)
        for ch in self._halves:
            done = torch.cuda.Event()
            done.record(ch["stream"])
            cur.wait_event(done)
        self._keep_conc = hold
        if sync:
            self.sync_concurrent()
        return out

    def sync_concurrent(self):
        for ch in (self._halves or []):
            ch["eng"].sync()
        self._keep_conc = None

    def sync(self):
        N.check(N.lib().wn_sync(self._h))
        self._keep = None
