#!/usr/bin/env python
"""A/B of two engine libraries on the full pass (development aid): bench.py runs alternated, and output parity.

Run (on an H100, from the repository root):
  python tools/ab_bench.py --base OTHER_LIB [--rounds 2 --pairs 5 --steps 50 --warmup 10] [--dump C3,C3MH,...] [--out DIR]
Each pair runs `bench.py --no-cpu-baseline --no-pack-leg --no-next-rows` once with OTHER_LIB and once with the in-tree library
(KR_ENGINE_LIB), in alternating order, and prints per run: ms per pass (`value`), the chain without the hash
(`pipeline_roofline.avg_ms`), k_match2 / k_decide2 / k_hash of the profiled pass and the two incremental legs.  --dump runs
`bench.py --dump-outputs` once per library and workload and compares every array.  The report and the dumps go under --out
(default: a new temporary directory), never into the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = os.path.join(ROOT, "kuberay_b200", "libkrengine.so")


def card() -> str:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def bench(lib: str, args: list[str]) -> dict:
    env = dict(os.environ, KR_ENGINE_LIB=lib)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", *args], capture_output=True, text=True, env=env, cwd=ROOT, timeout=900)
    if out.returncode != 0:
        raise RuntimeError(f"bench.py failed ({lib}):\n{out.stderr[-3000:]}")
    return json.loads(out.stdout.strip().splitlines()[-1])


def row(r: dict) -> dict:
    k = r["kernels_ms_per_step"]
    inc, loc = r["e2e_incremental_1pct_pod_churn"], r["e2e_incremental_1pct_of_clusters"]
    return {"ms_per_pass": r["ms_per_step"], "chain_ms": r["pipeline_roofline"]["avg_ms"], "k_match2": k.get("k_match2"), "k_decide2": k.get("k_decide2"),
            "k_hash": k.get("k_hash"), "inc_ms": inc["ms_per_step"], "inc_kernels_ms": inc["kernels_ms"], "loc_ms": loc["ms_per_step"],
            "loc_kernels_ms": loc["kernels_ms"], "sm_mhz": r["clocks"]["sm_mhz"], "reasons": r["clocks"]["reasons"]}


def fmt(x) -> str:
    return f"{x:8.4f}" if isinstance(x, float) else f"{x!s:>8}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, help="the other library (e.g. the parent commit's build)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--pairs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--dump", default="", help="comma-separated workloads whose outputs are compared")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    a.out = a.out or tempfile.mkdtemp(prefix="kr_ab_")
    os.makedirs(a.out, exist_ok=True)
    print("output:", a.out, flush=True)
    libs = {"base": os.path.abspath(a.base), "new": NEW}
    report = {"card_before": card(), "runs": []}
    print("card:", report["card_before"], flush=True)

    for wl in [w for w in a.dump.split(",") if w]:
        dirs = {}
        for name, lib in libs.items():
            dirs[name] = os.path.join(a.out, "dump", name, wl)
            bench(lib, ["--workload", wl, "--steps", "3", "--warmup", "3", "--no-cpu-baseline", "--no-pack-leg", "--no-next-rows", "--dump-outputs", dirs[name]])
        files = sorted(set(os.listdir(dirs["base"])) | set(os.listdir(dirs["new"])))
        bad = [f for f in files if not (os.path.exists(os.path.join(dirs["base"], f)) and os.path.exists(os.path.join(dirs["new"], f))
                                        and np.array_equal(np.load(os.path.join(dirs["base"], f)), np.load(os.path.join(dirs["new"], f))))]
        report[f"dump_{wl}"] = {"arrays": len(files), "different": bad}
        print(f"outputs {wl}: {len(files)} arrays, {'identical' if not bad else 'DIFFERENT: ' + ', '.join(bad)}", flush=True)

    cols = ["ms_per_pass", "chain_ms", "k_match2", "k_decide2", "k_hash", "inc_ms", "inc_kernels_ms", "loc_ms", "loc_kernels_ms", "sm_mhz"]
    print("round pair lib  " + " ".join(f"{c[:8]:>8}" for c in cols), flush=True)
    bargs = ["--steps", str(a.steps), "--warmup", str(a.warmup), "--no-cpu-baseline", "--no-pack-leg", "--no-next-rows"]
    for rnd in range(a.rounds):
        for p in range(a.pairs):
            order = ["base", "new"] if (rnd * a.pairs + p) % 2 == 0 else ["new", "base"]
            for name in order:
                r = row(bench(libs[name], bargs))
                report["runs"].append({"round": rnd, "pair": p, "lib": name, **r})
                print(f"{rnd:5d} {p:4d} {name:4s} " + " ".join(fmt(r[c]) for c in cols) + (f"  {r['reasons']}" if r["reasons"] else ""), flush=True)
    for rnd in range(a.rounds):
        b = [r["ms_per_pass"] for r in report["runs"] if r["round"] == rnd and r["lib"] == "base"]
        n = [r["ms_per_pass"] for r in report["runs"] if r["round"] == rnd and r["lib"] == "new"]
        print(f"round {rnd}: base {min(b):.4f}-{max(b):.4f} (median {np.median(b):.4f})  new {min(n):.4f}-{max(n):.4f} (median {np.median(n):.4f})  "
              f"every new run faster than every base run: {max(n) < min(b)}", flush=True)
    report["card_after"] = card()
    print("card:", report["card_after"], flush=True)
    with open(os.path.join(a.out, "report.json"), "w") as f:
        json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
