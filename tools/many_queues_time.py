"""Time the allocate cycle on a C3-shaped cluster (50 000 tasks, 5 000 PodGroups, 5 000 nodes) spread over Q queues, and the
shipped action list with its Running filler pods at a few Q.  Every result is checked bit-exactly against the CPU emulation.
    python tools/many_queues_time.py [--queues 1,8,64,300,1000,5000] [--cycle-queues 8,1000] [--reps 5] [--out FILE]
Prints one JSON object: the device, its power limit and SM clock, then per Q the load time, ms per kb_allocate (median and
spread over --reps cycles after one warm-up), kernel launches, whether the persistent pipeline ran, and the same for kb_cycle."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
from kube_batch_b200 import engine, synth
import util

ACTS = ("reclaim", "allocate", "backfill", "preempt")


def c3_with_queues(Q: int):
    spec = synth.CONFIGS["c3"]
    from dataclasses import replace
    s = synth.generate(replace(spec, name=f"c3q{Q}", queues=Q))
    return s, synth.config_conf("c3")


def device_info() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim, smax, scur = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": plim, "max_sm_clock": smax, "sm_clock_at_start": scur}
    except Exception as ex:                       # the numbers below still stand; say what is missing
        return {"gpu": "unknown", "error": str(ex)}


def time_calls(fn, reps: int):
    fn()                                          # warm-up: module load, graph capture
    ms, last = [], None
    for _ in range(reps):
        t0 = time.perf_counter(); last = fn(); ms.append(1e3 * (time.perf_counter() - t0))
    return ms, last


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queues", default="1,8,64,300,1000,5000")
    ap.add_argument("--cycle-queues", default="8,1000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    out = {"device": device_info(), "allocate": {}, "cycle": {}}
    eng = engine.Engine(0)
    for Q in [int(x) for x in a.queues.split(",") if x]:
        s, conf = c3_with_queues(Q)
        t0 = time.perf_counter(); eng.load(s, conf); load_ms = 1e3 * (time.perf_counter() - t0)
        ms, res = time_calls(eng.allocate, a.reps)
        ref = util.emu_allocate(s, conf, mode=1)
        st = res.stats
        out["allocate"][Q] = {"queues_with_jobs": int(len(np.unique(s.job_queue))), "load_ms": round(load_ms, 1),
                              "ms_median": round(float(np.median(ms)), 3), "ms_min": round(min(ms), 3), "ms_max": round(max(ms), 3),
                              "gpu_ms": round(float(st.gpu_ms), 3), "kernel_launches": int(st.kernel_launches), "pipeline": int(st.pipeline),
                              "visits": int(st.visits) if hasattr(st, "visits") else None,
                              "allocated": int((res.decisions["kind"] == 1).sum()),
                              "bit_exact_vs_emulation": bool((ref.decisions == res.decisions).all())}
        print(json.dumps({"allocate": Q, **out["allocate"][Q]}), flush=True)
    for Q in [int(x) for x in a.cycle_queues.split(",") if x]:
        s, conf = c3_with_queues(Q)
        run = synth.running_of(s, 0.3)
        eng.load(s, conf).load_running(run)
        ms, (res, ev, order, bounds) = time_calls(lambda: eng.cycle(ACTS), a.reps)
        g, gev, gorder = util.emu_cycle(s, conf, ACTS, run, mode=1)
        st = res.stats
        out["cycle"][Q] = {"running_pods": int(len(run["node"])), "ms_median": round(float(np.median(ms)), 3), "ms_min": round(min(ms), 3),
                           "ms_max": round(max(ms), 3), "gpu_ms": round(float(st.gpu_ms), 3), "kernel_launches": int(st.kernel_launches),
                           "evictions": int(ev.sum()),
                           "bit_exact_vs_emulation": bool((g.decisions == res.decisions).all() and (gev == ev).all() and (gorder == order).all())}
        print(json.dumps({"cycle": Q, **out["cycle"][Q]}), flush=True)
    eng.close()
    text = json.dumps(out, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)
    bad = [k for part in ("allocate", "cycle") for k, v in out[part].items() if not v["bit_exact_vs_emulation"]]
    if bad:
        sys.exit(f"not bit-exact: {bad}")


if __name__ == "__main__":
    main()
