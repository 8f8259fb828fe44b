"""Cost of per-step Weight normalisation on the generic window kernel: the DiehlAndCook2015 shape (Input(784) -> 1600
with inhibition, input Weight norm 78.4, MCC PostPre) with a 'sample' Weight and with a 'time step' Weight, both on
tier 1, at B = 1 and 128, T = 250.  Windows alternate between the two arms; the median of 7 windows per arm, timed with
CUDA events, is reported with the card's name and power limit read in the same run.  The per-step pass reads the input
weights twice (column sums, then the rescale) and writes them once: 3 * n_src * n_tgt * 4 bytes per step.

    python bench_weight_norm.py [--windows 7]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]

import torch  # noqa: E402


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    except Exception:   # (no nvidia-smi: the name from torch, the power limit unknown)
        name, power = torch.cuda.get_device_name(0), "unknown"
    return {"gpu": name, "power_limit": power}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_weight_norm.py needs a CUDA device"
    import cases
    import weight_norm_nets as wn

    ns = cases.namespace("b200")
    T, n_in, n = 250, 784, 1600
    out = {"bench": "weight_norm", "T": T, "n_src": n_in, "n_tgt": n, **card(), "results": []}
    for B in (1, 128):
        nets = {}
        for freq in ("sample", "time step"):
            net, x = wn.dc_graph(ns, B, freq, n_in=n_in, n=n, T=T)
            net.force_tier = 1
            net.to("cuda")
            nets[freq] = (net, x.cuda())
        times = {k: [] for k in nets}
        for it in range(args.windows + 1):   # window 0 of each arm warms up
            for freq, (net, x) in nets.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                net.run(inputs={"X": x}, time=T, one_spike_seed=it)
                e1.record()
                torch.cuda.synchronize()
                net.check_errors()
                if it:
                    times[freq].append(e0.elapsed_time(e1))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        added = med["time step"] - med["sample"]
        step_bytes = 3 * n_in * n * 4
        out["results"].append({"B": B, "sample_ms": round(med["sample"], 3), "time_step_ms": round(med["time step"], 3),
                               "ratio": round(med["time step"] / med["sample"], 3), "added_ms": round(added, 3),
                               "bytes_per_step": step_bytes,
                               "implied_GBps": round(step_bytes * T / (added * 1e-3) / 1e9, 1) if added > 0 else None})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
