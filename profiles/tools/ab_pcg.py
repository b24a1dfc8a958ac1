"""A/B of the cooperative k_cg_step against the four-kernel PCG chain on the C3 timed loop of bench.py: alternating
I3D_PCG_FUSED=1 / 0 runs (one process each), the GN iteration rate, the pcg phase, the per-kernel table of the untimed detail step and
the per-step PCG iteration counts, with the card's name and power limit read in the same call.

    python profiles/tools/ab_pcg.py [--runs 3] [--steps 30] [--warmup 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as ex:          # the tool still reports the timings
        return f"unknown ({ex})"


def run(fused, steps, warmup):
    env = dict(os.environ, I3D_PCG_FUSED="1" if fused else "0")
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--no-cpu-baseline", "--no-parity-check", "--no-e2e", "--no-lighting"]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    if out.returncode != 0:
        raise RuntimeError(f"bench.py (I3D_PCG_FUSED={int(fused)}) failed:\n{out.stderr[-3000:]}")
    line = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])
    ps = line["per_step"]
    pcg = ps["phase_ms"]["pcg"]
    return {"value": line["value"], "pcg_ms_mean": sum(pcg) / len(pcg), "total_ms_mean": sum(ps["phase_ms"]["total"]) / len(pcg),
            "cg_iterations": ps["cg_iterations"], "kernel_ms_detail_step": ps["kernel_ms_detail_step"]}


def summary(rs):
    v = [r["value"] for r in rs]
    p = [r["pcg_ms_mean"] for r in rs]
    mean = sum(v) / len(v)
    return {"value_mean": mean, "value_min": min(v), "value_max": max(v), "value_spread_pct": 100.0 * (max(v) - min(v)) / mean,
            "pcg_ms_mean": sum(p) / len(p), "pcg_ms_min": min(p), "pcg_ms_max": max(p)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"fused": [], "chain": []}
    for i in range(a.runs):
        for fused in ((True, False) if i % 2 == 0 else (False, True)):
            r = run(fused, a.steps, a.warmup)
            res["fused" if fused else "chain"].append(r)
            print(("fused" if fused else "chain"), f"{r['value']:.2f} GN iter/s, pcg {r['pcg_ms_mean']:.3f} ms", flush=True)
    sf, sc = summary(res["fused"]), summary(res["chain"])
    report = {
        "card": card(), "workload": "c3", "steps": a.steps, "warmup": a.warmup, "runs_per_arm": a.runs,
        "fused": sf, "chain": sc,
        "value_gain_pct": 100.0 * (sf["value_mean"] / sc["value_mean"] - 1.0),
        "pcg_reduction_pct": 100.0 * (1.0 - sf["pcg_ms_mean"] / sc["pcg_ms_mean"]),
        "ranges_overlap": not (sf["value_min"] > sc["value_max"] or sc["value_min"] > sf["value_max"]),
        "cg_iterations_identical": all(r["cg_iterations"] == res["chain"][0]["cg_iterations"] for r in res["fused"] + res["chain"]),
        "cg_iterations": res["chain"][0]["cg_iterations"],
        "kernel_ms_detail_step": {"fused": res["fused"][0]["kernel_ms_detail_step"], "chain": res["chain"][0]["kernel_ms_detail_step"]},
        "runs": res,
    }
    print(json.dumps({k: v for k, v in report.items() if k != "runs"}, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
