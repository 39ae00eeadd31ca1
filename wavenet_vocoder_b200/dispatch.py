# coding: utf-8
"""Directory-level synthesis: the part of the reference's ``evaluate.py`` that sits either side of
the hot path (SURVEY.md 8(f-2), 8(f-3)) -- read ``*-feats.npy`` mel files, batch them, synthesise,
decode and write 16-bit wav files -- re-organised for the engine:

* the reference pads every utterance of a DataLoader batch to the longest one and loops batches on one
  device (evaluate.py:50-58, :162-204).  Here utterances are sharded over ranks by total length
  (``parallel.shard_utterances``) and, inside a rank, sorted by length and grouped into launches of at
  most ``tile`` utterances, so the padding inside a launch is small;
* decode follows synthesis.py:66-84 / evaluate.py:215-251 -- class ids -> inverse mu-law, optional inverse
  pre-emphasis, gain, trim to the utterance's own length, clip, int16 -- as one device kernel of libwn
  (``decode_device``; csrc/wn_aux.cuh) writing int16 directly.

File formats are the reference's: ``<name>-feats.npy`` = (frames, num_mels) float32 written by
``datasets/wavallin.py`` (np.save, :104-107); output ``<name>_gen.wav`` (evaluate.py:229-231).
"""
from __future__ import annotations

import os
from glob import glob
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from .parallel import shard_utterances, tile_batches


INPUT_TYPES = {"raw": 0, "mulaw": 1, "mulaw-quantize": 2}


def decode_device(y_hat: torch.Tensor, lengths: Optional[Sequence[int]] = None, input_type: str = "raw",
                  quantize_channels: int = 65536, postprocess: Optional[str] = None,
                  global_gain_scale: float = 0.0, preemphasis_coef: float = 0.85, want_float: bool = False):
    """Model output (B,C,T) on the GPU -> int16 waveforms (B,T) on the GPU (and, optionally, the float waveforms
    ``batch_wavegen`` returns), in ONE kernel of libwn (csrc/wn_aux.cuh): inverse mu-law for "mulaw" /
    "mulaw-quantize" (synthesis.py:66-74), inv_preemphasis when ``postprocess == "inv_preemphasis"``
    (synthesis.py:76-78, audio.py:57-58), division by ``global_gain_scale`` (synthesis.py:80-82), trim to
    ``lengths`` (zeros beyond), clip and int16 (evaluate.py:215,247,43-48).  No CPU path: raises off the GPU."""
    import ctypes as C
    from . import _native as N
    if y_hat.device.type != "cuda":
        raise RuntimeError("decode_device runs on a CUDA tensor only (no CPU fallback)")
    if postprocess not in (None, "", "none", "inv_preemphasis"):
        raise ValueError("unsupported postprocess %r" % (postprocess,))
    B = y_hat.size(0)
    kind = INPUT_TYPES[input_type]
    y_s = y_i = None
    if kind == 2:
        y_i = y_hat.max(1)[1].view(B, -1).to(torch.int32).contiguous()          # synthesis.py:68
        T = y_i.size(1)
    else:
        y_s = y_hat.reshape(B, -1).float().contiguous()
        T = y_s.size(1)
    dev = y_hat.device
    len_t = None if lengths is None else torch.tensor([int(v) for v in lengths], dtype=torch.int32, device=dev)
    pcm = torch.empty(B, T, dtype=torch.int16, device=dev)
    flt = torch.empty(B, T, dtype=torch.float32, device=dev) if want_float else None
    coef = float(preemphasis_coef) if postprocess == "inv_preemphasis" else 0.0
    with torch.cuda.device(dev):
        N.check(N.lib().wn_decode(None if y_s is None else y_s.data_ptr(), None if y_i is None else y_i.data_ptr(), B, T,
                                  None if len_t is None else len_t.data_ptr(), kind, int(quantize_channels),
                                  C.c_float(coef), C.c_float(float(global_gain_scale)),
                                  None if flt is None else flt.data_ptr(), pcm.data_ptr(),
                                  torch.cuda.current_stream(dev).cuda_stream))
    return (pcm, flt) if want_float else pcm


class StreamDecoder:
    """``decode_device`` chunk by chunk: feed consecutive chunks (B,C,T_i) of the model output and get each chunk's
    int16 (and, with ``want_float``, float) waveform; the concatenation equals one ``decode_device`` call over the
    whole output bit for bit.  The inv_preemphasis recursion carries over chunk boundaries on the device
    (wn_decode_stream); ``lengths`` are the utterances' lengths in the whole output."""

    def __init__(self, B: int, device, input_type: str = "raw", quantize_channels: int = 65536,
                 postprocess: Optional[str] = None, global_gain_scale: float = 0.0, preemphasis_coef: float = 0.85,
                 lengths: Optional[Sequence[int]] = None, want_float: bool = False):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("StreamDecoder runs on a CUDA device only (no CPU fallback)")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if postprocess not in (None, "", "none", "inv_preemphasis"):
            raise ValueError("unsupported postprocess %r" % (postprocess,))
        self.B, self.device = int(B), device
        self.kind = INPUT_TYPES[input_type]
        self.quantize_channels = int(quantize_channels)
        self.coef = float(preemphasis_coef) if postprocess == "inv_preemphasis" else 0.0
        self.gain = float(global_gain_scale)
        self.lengths = None if lengths is None else [int(v) for v in lengths]
        self.want_float = bool(want_float)
        self.carry = torch.zeros(self.B, dtype=torch.float32, device=device)   # coef * last sample of the previous chunk
        self.t = 0

    def __call__(self, y_hat: torch.Tensor):
        import ctypes as C
        from . import _native as N
        B = self.B
        if y_hat.device != self.device or y_hat.size(0) != B:
            raise ValueError("expected a (%d,C,T) chunk on %s" % (B, self.device))
        y_s = y_i = None
        if self.kind == 2:
            y_i = y_hat.max(1)[1].view(B, -1).to(torch.int32).contiguous()      # synthesis.py:68
            T = y_i.size(1)
        else:
            y_s = y_hat.reshape(B, -1).float().contiguous()
            T = y_s.size(1)
        pcm = torch.empty(B, T, dtype=torch.int16, device=self.device)
        flt = torch.empty(B, T, dtype=torch.float32, device=self.device) if self.want_float else None
        if T == 0:
            return (pcm, flt) if self.want_float else pcm
        len_t = None
        if self.lengths is not None:
            len_t = torch.tensor([max(0, v - self.t) for v in self.lengths], dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            N.check(N.lib().wn_decode_stream(None if y_s is None else y_s.data_ptr(), None if y_i is None else y_i.data_ptr(),
                                             B, T, None if len_t is None else len_t.data_ptr(), self.kind,
                                             self.quantize_channels, C.c_float(self.coef), C.c_float(self.gain),
                                             None if flt is None else flt.data_ptr(), pcm.data_ptr(), self.carry.data_ptr(),
                                             torch.cuda.current_stream(self.device).cuda_stream))
        self.t += T
        return (pcm, flt) if self.want_float else pcm


def list_feature_files(data_dir: str) -> List[str]:
    files = sorted(glob(os.path.join(data_dir, "*-feats.npy")))
    if not files:
        raise FileNotFoundError("no *-feats.npy under %s" % data_dir)
    return files


def collate(feats: Sequence[np.ndarray], cin_pad: int) -> torch.Tensor:
    """(frames_i, D) arrays -> (B, D, max_frames + 2*cin_pad): zero padded to the longest (evaluate.py:50-58)
    then edge-replicated by cin_pad on both sides (evaluate.py:163-164)."""
    max_len = max(f.shape[0] for f in feats)
    D = feats[0].shape[1]
    c = np.zeros((len(feats), max_len, D), dtype=np.float32)
    for i, f in enumerate(feats):
        c[i, :f.shape[0]] = f
    ct = torch.from_numpy(c).transpose(1, 2).contiguous()
    if cin_pad > 0:
        ct = F.pad(ct, (cin_pad, cin_pad), mode="replicate")
    return ct


def synthesize_directory(model, data_dir: str, dst_dir: str, *, hop_size: int, cin_pad: int = 0,
                         sample_rate: int = 22050, tile: int = 4, rank: int = 0, world: int = 1,
                         input_type: str = "raw", quantize_channels: int = 65536,
                         postprocess: Optional[str] = None, global_gain_scale: float = 0.0,
                         synth: Optional[Callable[[torch.Tensor, int], torch.Tensor]] = None,
                         decode: Optional[Callable] = None, write: bool = True) -> Dict[str, np.ndarray]:
    """Synthesise this rank's share of ``data_dir`` and write ``<name>_gen.wav`` into ``dst_dir``.
    ``synth(c, T)`` defaults to ``model.incremental_forward(c=c, T=T)`` (c: (B, D, frames + 2*cin_pad));
    ``decode(y_hat, lengths) -> (B,T) int16`` defaults to the device kernel (``decode_device``).  Both hooks exist
    for the host-logic tests, which run without a GPU.  Returns {name: int16 waveform} for this rank's utterances."""
    from scipy.io import wavfile
    files = list_feature_files(data_dir)
    feats = [np.load(f).astype(np.float32) for f in files]
    lengths = [f.shape[0] * hop_size for f in feats]
    mine = shard_utterances(lengths, world)[rank]
    if synth is None:
        def synth(c, T):
            with torch.no_grad():
                return model.incremental_forward(c=c, T=T)
    if decode is None:
        def decode(y_hat, lens):
            return decode_device(y_hat, lens, input_type, quantize_channels, postprocess, global_gain_scale)
    if write:
        os.makedirs(dst_dir, exist_ok=True)
    results: Dict[str, np.ndarray] = {}
    for launch in tile_batches(mine, lengths, tile):
        c = collate([feats[i] for i in launch], cin_pad)
        T = (c.shape[-1] - 2 * cin_pad) * hop_size
        pcm_all = decode(synth(c, T), [lengths[i] for i in launch])
        pcm_all = pcm_all.cpu().numpy() if isinstance(pcm_all, torch.Tensor) else np.asarray(pcm_all)
        for row, i in enumerate(launch):
            pcm = pcm_all[row][:lengths[i]].astype(np.int16)            # trim the batch padding (evaluate.py:215)
            name = os.path.splitext(os.path.basename(files[i]))[0].replace("-feats", "")
            results[name] = pcm
            if write:
                wavfile.write(os.path.join(dst_dir, "%s_gen.wav" % name), sample_rate, pcm)
    return results
