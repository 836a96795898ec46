"""Milliseconds per denoise step of the config-2 and config-3 workloads of bench.py at the square frame sizes of the
reference web UI's resolution slider (256..512 in steps of 64).  Prints one JSON line with the card's name and power
limit, read in the same run.

    python tools/bench_resolutions.py [--steps K] [--warmup W] [--res 256,320,384,448,512] [--workloads config2,config3]

Each cell builds ``bench.Workload(res=...)`` (N = 8 keyframes, CFG => 16 samples, eager execution) and walks the
15-step schedule from its start: W warm-up steps, then K timed steps between CUDA events on the current stream.
At 320, 384 and 448 decoder layer 0 (and at 320 and 448 layer 1) has a token count that is not a multiple of 8, so config 3's
Gram-L1 loss runs on the ragged kernels there (DESIGN §3.2).  Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                              "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [f.strip() for f in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:                               # the card name from torch, the limit unknown
        return {"name": torch.cuda.get_device_name(), "power_limit": "unavailable (%s)" % type(e).__name__}


def time_steps(wl, steps, warmup):
    for k in range(warmup):
        wl.step(k)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for k in range(warmup, warmup + steps):
        wl.step(k)
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=15, help="timed steps (15 = one walk of the schedule)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--res", default="256,320,384,448,512")
    ap.add_argument("--workloads", default="config2,config3")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resolutions: needs a CUDA device")
    device = torch.device("cuda", 0)
    result = {"metric": "ms per denoise step", "frames": bench.N_FRAMES, "card": card(), "ms_per_step": {}}
    for workload in args.workloads.split(","):
        if workload not in ("config2", "config3"):
            raise SystemExit("bench_resolutions: unknown workload %r" % workload)
        row = {}
        for res in (int(r) for r in args.res.split(",")):
            opt = workload == "config3"
            wl = bench.Workload(device, seed=0, res=res, optimise=opt, with_gmflow=opt)
            row["%dx%d" % (res, res)] = round(time_steps(wl, args.steps, args.warmup), 2)
            del wl
            torch.cuda.empty_cache()
        result["ms_per_step"][workload] = row
    print(json.dumps(result))


if __name__ == "__main__":
    main()
