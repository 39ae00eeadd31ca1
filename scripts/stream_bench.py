# coding: utf-8
"""Streaming synthesis on BASELINE config 2 (MoL, 24 layers, 512/512/256, 80 mel channels, B=1, T=22050): one
wn_generate call against the same utterance made through wn_stream_generate, in one chunk and in chunks of 256 / 1024 /
4096 samples, each chunk synchronised as a streaming consumer would.  Prints, per mode, samples/s, the time to the
first chunk and the cost of one chunk boundary ((chunked - one chunk) / boundaries; the stream kernel is a separate
instantiation, so its per-step cost is the one-chunk mode against the one-shot call), medians of --runs runs, and the
card's name and power limit (nvidia-smi, read only).

--B 8 --engine 7 makes 8 utterances at once: one engine-7 wn_generate, and one engine-7 stream of 8 (on an engine-7
handle of the same weights).  --engine 5 with B > 4 runs the one-shot call as wn_generate's consecutive tiles of 4 and
the stream as streams of at most 4 called in turn, each chunk synchronised; the time to the first chunk is then the
time until every utterance has its first chunk.  --engine 5,7 alternates the two engines run by run in one process.

    python scripts/stream_bench.py [--T 22050] [--runs 3] [--chunks 256,1024,4096] [--B 1] [--engine 5]
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
    ap.add_argument("--B", type=int, default=1, help="utterances")
    ap.add_argument("--engine", default="5", help="5, 7 or 5,7 (alternated run by run)")
    args = ap.parse_args()
    engines = [int(e) for e in args.engine.split(",")]
    assert engines and set(engines) <= {5, 7}, args.engine
    B = args.B
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
    mel = torch.randn(B, 80, frames, generator=torch.Generator().manual_seed(1)).to(dev)
    c = eng.upsample(mel, eng.upsampled_length(frames))[:, :T].contiguous()     # (B,T,80) sample-rate conditioning
    handle = {5: eng, 7: eng.engine7() if 7 in engines else None}

    def one_shot(e, seed):
        t0 = time.perf_counter()
        y, _ = handle[e].generate(B=B, T=T, c=c, seed=seed)
        t1 = time.perf_counter()
        return t1 - t0, t1 - t0, y

    def chunked(e, n, seed):
        tile = B if e == 7 else 4              # engine 5: streams of at most 4 rows, row b draws row b's noise
        streams = [(handle[e].open_stream(B=min(tile, B - b0), seed=seed, philox_row0=b0, engine=e), b0)
                   for b0 in range(0, B, tile)]
        ys, first = [[] for _ in streams], None
        t0 = time.perf_counter()
        for t in range(0, T, n):
            k = min(n, T - t)
            for (s, b0), yk in zip(streams, ys):
                y, _ = s.generate(k, c=c[b0:b0 + s.B, t:t + k])      # synchronised: the chunk is ready when this returns
                yk.append(y)
            if first is None:
                first = time.perf_counter() - t0
        total = time.perf_counter() - t0
        for s, _ in streams:
            s.close()
        return total, first, torch.cat([torch.cat(yk, -1) for yk in ys], 0)

    modes = [("one_shot", None), ("stream_one_chunk", T)] + [("chunk_%d" % int(n), int(n)) for n in args.chunks.split(",")]
    res = {e: {} for e in engines}
    ref = {}
    for name, n in modes:
        tot, fst = {e: [] for e in engines}, {e: [] for e in engines}
        for e in engines:
            (one_shot(e, 7) if n is None else chunked(e, n, 7))       # warm-up
        for r in range(args.runs):
            for e in engines:
                a, b, y = one_shot(e, 7) if n is None else chunked(e, n, 7)
                tot[e].append(a), fst[e].append(b)
                if e not in ref:
                    ref[e] = y
                assert torch.equal(y, ref[e]), "%s engine %d: chunked output differs from one shot" % (name, e)
        for e in engines:
            tot[e].sort(), fst[e].sort()
            res[e][name] = dict(chunk=n, seconds=tot[e][len(tot[e]) // 2], samples_per_s=B * T / tot[e][len(tot[e]) // 2],
                                first_chunk_ms=1e3 * fst[e][len(fst[e]) // 2], runs=tot[e])
    for e in engines:
        one, whole = res[e]["one_shot"]["seconds"], res[e]["stream_one_chunk"]["seconds"]
        res[e]["stream_one_chunk"]["us_per_step_vs_one_shot"] = 1e6 * (whole - one) / T
        for name, n in modes[2:]:
            b = -(-T // n) - 1
            res[e][name]["boundaries"] = b
            res[e][name]["us_per_boundary"] = 1e6 * (res[e][name]["seconds"] - whole) / b
            res[e][name]["vs_one_shot"] = res[e][name]["seconds"] / one
    if engines == [5]:
        print(json.dumps(dict(card=card(), T=T, config="cfg2 B=%d" % B, modes=res[5]), indent=1))
    else:
        print(json.dumps(dict(card=card(), T=T, config="cfg2 B=%d" % B, engines=res), indent=1))


if __name__ == "__main__":
    main()
