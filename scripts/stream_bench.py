# coding: utf-8
"""Streaming synthesis on BASELINE config 2 (MoL, 24 layers, 512/512/256, 80 mel channels, B=1, T=22050): one
wn_generate call against the same utterance made through wn_stream_generate, in one chunk and in chunks of 256 / 1024 /
4096 samples, each chunk synchronised as a streaming consumer would.  Prints, per mode, samples/s, the time to the
first chunk and the cost of one chunk boundary ((chunked - one chunk) / boundaries; the stream kernel is a separate
instantiation, so its per-step cost is the one-chunk mode against the one-shot call), medians of --runs runs, and the
card's name and power limit (nvidia-smi, read only).

    python scripts/stream_bench.py [--T 22050] [--runs 3] [--chunks 256,1024,4096]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

CFG2 = dict(out_channels=30, layers=24, stacks=4, residual_channels=512, gate_channels=512,
            skip_out_channels=256, cin_channels=80, cin_pad=2, gin_channels=-1, scalar_input=True,
            output_distribution="Logistic", dropout=0.0, upsample_conditional_features=True,
            upsample_params={"upsample_scales": [4, 4, 4, 4], "cin_channels": 80, "cin_pad": 2})


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=22050)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--chunks", default="256,1024,4096")
    args = ap.parse_args()
    from wavenet_vocoder_b200 import WaveNet
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    m = WaveNet(**CFG2).eval()
    with torch.no_grad():
        m.last_conv_layers[3].bias[20:] -= 3.0
    m = m.to(dev)
    eng = m._get_engine()
    T = args.T
    frames = -(-T // 256) + 4
    mel = torch.randn(1, 80, frames, generator=torch.Generator().manual_seed(1)).to(dev)
    c = eng.upsample(mel, eng.upsampled_length(frames))[:, :T].contiguous()     # (1,T,80) sample-rate conditioning

    def one_shot(seed):
        t0 = time.perf_counter()
        y, _ = eng.generate(B=1, T=T, c=c, seed=seed)
        t1 = time.perf_counter()
        return t1 - t0, t1 - t0, y

    def chunked(n, seed):
        s = eng.open_stream(B=1, seed=seed)
        ys, first = [], None
        t0 = time.perf_counter()
        for t in range(0, T, n):
            k = min(n, T - t)
            y, _ = s.generate(k, c=c[:, t:t + k])      # synchronised: the chunk is ready when this returns
            ys.append(y)
            if first is None:
                first = time.perf_counter() - t0
        total = time.perf_counter() - t0
        s.close()
        return total, first, torch.cat(ys, -1)

    modes = [("one_shot", None), ("stream_one_chunk", T)] + [("chunk_%d" % int(n), int(n)) for n in args.chunks.split(",")]
    res = {}
    ref = None
    for name, n in modes:
        fn = one_shot if n is None else (lambda seed, n=n: chunked(n, seed))
        fn(7)                                           # warm-up
        tot, fst = [], []
        for r in range(args.runs):
            a, b, y = fn(7)
            tot.append(a), fst.append(b)
            if ref is None:
                ref = y
            assert torch.equal(y, ref), name + ": chunked output differs from one shot"
        tot.sort(), fst.sort()
        res[name] = dict(chunk=n, seconds=tot[len(tot) // 2], samples_per_s=T / tot[len(tot) // 2],
                         first_chunk_ms=1e3 * fst[len(fst) // 2], runs=tot)
    one, whole = res["one_shot"]["seconds"], res["stream_one_chunk"]["seconds"]
    res["stream_one_chunk"]["us_per_step_vs_one_shot"] = 1e6 * (whole - one) / T
    for name, n in modes[2:]:
        b = -(-T // n) - 1
        res[name]["boundaries"] = b
        res[name]["us_per_boundary"] = 1e6 * (res[name]["seconds"] - whole) / b
        res[name]["vs_one_shot"] = res[name]["seconds"] / one
    print(json.dumps(dict(card=card(), T=T, config="cfg2 B=1", modes=res), indent=1))


if __name__ == "__main__":
    main()
