# coding: utf-8
"""Teacher-forced scoring speed: wn_forward (csrc/wn_dense.cuh) against the PyTorch forward() of the same module, on
BASELINE config 2 (MoL, 24 layers, 512/512/256, 80 conditioning channels) at B = 1 and 8 with T = 22 050 and config 5
(MoL, 30 layers, 256/512/256) at B = 1 with T = 240 000, and one teacher-forced incremental_forward(return_params=True)
of config 2 at B = 1 (the per-step engine computing the same head outputs).

Every time is the median of --runs calls after --warmup calls, measured with CUDA events.  Achieved TFLOP/s uses the
FLOP of the model's multiply-accumulates computed from its shapes (2 x MAC per sample), against the H100 SXM data
sheet's 67 TFLOP/s FP32 bound and the 165 TFLOP/s 3xTF32 bound (495 TF32 / 3); the line names the bound that applies to
the arithmetic of that path (the PyTorch default mode runs cuDNN convolutions in TF32: 495).  The card's name and power
limit are read in the same run.

    python scripts/forward_bench.py [--runs 5] [--warmup 2]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

CONFIGS = {
    "cfg2": dict(out_channels=30, layers=24, stacks=4, residual_channels=512, gate_channels=512,
                 skip_out_channels=256, cin_channels=80, gin_channels=-1, scalar_input=True,
                 output_distribution="Logistic", dropout=0.0),
    "cfg5": dict(out_channels=30, layers=30, stacks=3, residual_channels=256, gate_channels=512,
                 skip_out_channels=256, cin_channels=80, gin_channels=-1, scalar_input=True,
                 output_distribution="Logistic", dropout=0.0),
}
RUNS = [("cfg2", 1, 22050), ("cfg2", 8, 22050), ("cfg5", 1, 240000)]
FP32_TFLOPS, TF32X3_TFLOPS, TF32_TFLOPS = 67.0, 495.0 / 3, 495.0


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def flop_per_sample(kw, kernel_size=3):
    R, G, S, O = kw["residual_channels"], kw["gate_channels"], kw["skip_out_channels"], kw["out_channels"]
    C = max(kw["cin_channels"], 0)
    first = R if kw["scalar_input"] else R * O
    mac = first + kw["layers"] * (G * (kernel_size * R + C) + (R + S) * (G // 2)) + S * S + O * S
    return 2 * mac


def timed(fn, runs, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("forward_bench.py measures on a CUDA device; none is visible")
    from wavenet_vocoder_b200 import WaveNet
    dev = torch.device("cuda", 0)
    print("card: %s" % card())
    results = []
    for name, B, T in RUNS:
        kw = CONFIGS[name]
        torch.manual_seed(0)
        m = WaveNet(**kw).eval()
        with torch.no_grad():
            m.last_conv_layers[3].bias[20:] -= 3.0
        m = m.to(dev)
        gen = torch.Generator().manual_seed(1)
        x = ((torch.rand(B, 1, T, generator=gen) * 2 - 1) * 0.8).to(dev)
        c = torch.randn(B, kw["cin_channels"], T, generator=gen).to(dev)
        eng = m._get_engine()
        xs, ct = x[:, 0, :].contiguous(), c.transpose(1, 2).contiguous()
        flop = flop_per_sample(kw) * B * T
        row = dict(config=name, B=B, T=T, gflop=round(flop / 1e9, 1))

        t_native = timed(lambda: eng.forward(test_scalar=xs, c=ct, sync=False), args.runs, args.warmup)
        eng.sync()
        native = eng.forward(test_scalar=xs, c=ct)
        row["wn_forward"] = dict(s=t_native, samples_per_s=B * T / t_native, tflops=flop / t_native / 1e12,
                                 bound="3xTF32 %.0f" % TF32X3_TFLOPS, share=flop / t_native / 1e12 / TF32X3_TFLOPS)
        cudnn, mm = torch.backends.cudnn, torch.backends.cuda.matmul
        saved = (cudnn.allow_tf32, mm.allow_tf32)
        for mode, tf32, bound in (("torch_fp32", False, FP32_TFLOPS), ("torch_default", saved[0], TF32_TFLOPS)):
            cudnn.allow_tf32, mm.allow_tf32 = tf32, tf32 and saved[1]
            with torch.no_grad():
                t = timed(lambda: m(x, c=c, softmax=False), args.runs, args.warmup)
                ref = m(x, c=c, softmax=False)
            row[mode] = dict(s=t, samples_per_s=B * T / t, tflops=flop / t / 1e12,
                             bound=("FP32 %.0f" if bound == FP32_TFLOPS else "TF32 %.0f") % bound,
                             share=flop / t / 1e12 / bound, max_abs_diff_to_wn_forward=float((ref - native).abs().max()))
            del ref
        cudnn.allow_tf32, mm.allow_tf32 = saved
        if (name, B) == ("cfg2", 1):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, p = m.incremental_forward(test_inputs=x, c=c, T=T, seed=1, return_params=True)
            torch.cuda.synchronize()
            t = time.perf_counter() - t0
            row["incremental_forward_teacher_forced"] = dict(s=t, samples_per_s=B * T / t,
                                                             max_abs_diff_to_wn_forward=float((p - native).abs().max()))
        results.append(row)
        print(json.dumps(row))
        del m, eng, native
        torch.cuda.empty_cache()
    print("\n%-5s %2s %7s | %-28s | %-28s | %-28s" % ("cfg", "B", "T", "wn_forward (3xTF32)", "torch fp32 (IEEE)",
                                                    "torch default (TF32)"))
    for r in results:
        cells = []
        for k in ("wn_forward", "torch_fp32", "torch_default"):
            v = r[k]
            cells.append("%8.2f ms %6.1f TF/s %4.0f%%" % (v["s"] * 1e3, v["tflops"], 100 * v["share"]))
        print("%-5s %2d %7d | %s | %s | %s" % (r["config"], r["B"], r["T"], *cells))
        if "incremental_forward_teacher_forced" in r:
            v = r["incremental_forward_teacher_forced"]
            print("      incremental_forward(return_params=True), same utterance: %.3f s (%.0f samples/s)" % (
                v["s"], v["samples_per_s"]))
    print("card: %s" % card())


if __name__ == "__main__":
    main()
