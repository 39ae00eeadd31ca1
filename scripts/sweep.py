# coding: utf-8
"""Timing sweeps of the synthesis kernel on one GPU.  Each variant runs in a fresh process because
the planner reads its tuning knobs (WN_NUM_CTAS, WN_NCOPY, WN_RING_SLOTS, WN_RESIDENT, ...) from the
environment.   python scripts/sweep.py cfg2:T=4000 cfg2:T=4000,WN_RING_SLOTS=6,WN_RESIDENT=0 ..."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CFGS = {
    "cfg1": dict(out_channels=256, layers=12, stacks=2, residual_channels=64, gate_channels=128,
                 skip_out_channels=64, cin_channels=-1, gin_channels=-1, scalar_input=False, dropout=0.0),
    "cfg2": dict(out_channels=30, layers=24, stacks=4, residual_channels=512, gate_channels=512,
                 skip_out_channels=256, cin_channels=80, gin_channels=-1, scalar_input=True,
                 output_distribution="Logistic", dropout=0.0),
    "cfg3": dict(out_channels=2, layers=24, stacks=4, residual_channels=128, gate_channels=256,
                 skip_out_channels=128, cin_channels=80, gin_channels=16, n_speakers=16,
                 use_speaker_embedding=True, scalar_input=True, output_distribution="Normal", dropout=0.0),
    "cfg5": dict(out_channels=30, layers=30, stacks=3, residual_channels=256, gate_channels=512,
                 skip_out_channels=256, cin_channels=80, gin_channels=-1, scalar_input=True,
                 output_distribution="Logistic", dropout=0.0),
    # config 2 without local conditioning (isolates the conditioning warp)
    "cfg2nc": dict(out_channels=30, layers=24, stacks=4, residual_channels=512, gate_channels=512,
                   skip_out_channels=256, cin_channels=-1, gin_channels=-1, scalar_input=True,
                   output_distribution="Logistic", dropout=0.0),
}


def child(name, T, B, reps):
    import torch
    from wavenet_vocoder_b200 import WaveNet
    kw = CFGS[name]
    torch.manual_seed(0)
    m = WaveNet(**kw).eval()
    with torch.no_grad():
        if kw["scalar_input"]:
            O = kw["out_channels"]
            b = m.last_conv_layers[3].bias
            if O == 2:
                b[1] -= 3.0
            else:
                b[2 * (O // 3):] -= 3.0
    m = m.cuda()
    eng = m._get_engine()
    C = max(kw["cin_channels"], 0)
    c = torch.randn(B, T, C, device="cuda") if C else None
    g = torch.randn(B, kw["gin_channels"], device="cuda") * 0.1 if kw["gin_channels"] > 0 else None
    best = 1e30
    for i in range(reps + 1):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.generate(B=B, T=T, c=c, g=g, seed=i, sync=False)
        e1.record()
        eng.sync()
        if i > 0:
            best = min(best, e0.elapsed_time(e1))
    plan = eng.plan(B)
    print(json.dumps(dict(us_per_step=best * 1e3 / T, samples_per_s=B * T / (best * 1e-3),
                          P=plan["num_ctas"], BT=plan["batch_tile"], res=plan["resident_blobs"],
                          ring=plan["ring_slots"], ncopy=plan["exchange_copies"], smem=plan["smem_bytes"],
                          rings_smem=plan["rings_in_smem"])))


def main():
    if sys.argv[1] == "--child":
        child(sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]))
        return
    for spec in sys.argv[1:]:
        name, _, rest = spec.partition(":")
        env = dict(os.environ)
        T, B, reps = 2000, 1, 2
        for kv in filter(None, rest.split(",")):
            k, v = kv.split("=")
            if k == "T":
                T = int(v)
            elif k == "B":
                B = int(v)
            elif k == "reps":
                reps = int(v)
            else:
                env[k] = v
        r = subprocess.run([sys.executable, __file__, "--child", name, str(T), str(B), str(reps)], env=env,
                           capture_output=True, text=True, timeout=600)
        out = r.stdout.strip().splitlines()
        print("%-60s %s" % (spec, out[-1] if out and r.returncode == 0 else "FAILED rc=%d %s" % (r.returncode, r.stderr[-300:])))
        for ln in r.stderr.splitlines():
            if ln.startswith("WN_PROF") and not ln.startswith("WN_PROF_BLOCK"):   # scripts/stage_prof.py reads those
                print("    " + ln)
        sys.stdout.flush()


if __name__ == "__main__":
    main()
