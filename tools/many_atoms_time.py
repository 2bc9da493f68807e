"""ms per cycle of one seeded cluster at W = 2 and 4 (the 4-word kernel instances; W = 2 may take the persistent pipeline) and at
W = 8 and 16 (the wide-atom instances): kb_allocate and the shipped action list, median of several cycles after a warm-up, each
checked against the emulation with wide-atom class records.

    python tools/many_atoms_time.py [--tasks 20000] [--nodes 2000] [--reps 5]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from kube_batch_b200 import engine, synth  # noqa: E402
from kube_batch_b200.snapshot import PluginConf  # noqa: E402
import util  # noqa: E402

FULL_LIST = ("reclaim", "allocate", "backfill", "preempt")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tasks", type=int, default=20000)
    ap.add_argument("--nodes", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    wide = C.CDLL(os.path.join(ROOT, "tests", "emu_wide_atoms", "libkbemu_wide_atoms.so"))
    wide.kbemu_last_error.restype = C.c_char_p
    conf = PluginConf.default()
    eng = engine.Engine(0)
    out = {"gpu": smi, "tasks": a.tasks, "nodes": a.nodes, "rows": []}
    for W in (2, 4, 8, 16):
        s = synth.random_session(11, tasks=a.tasks, jobs=a.tasks // 10, nodes=a.nodes, queues=4, oversub=2.0, W=W)
        run = synth.running_of(s, 0.4)
        eng.load(s, conf).load_running(run)
        util._emu = wide                                               # the emulation with 16-word class records
        ref = util.emu_allocate(s, conf, mode=1)
        e, eev, eorder = util.emu_cycle(s, conf, FULL_LIST, run, mode=1)
        t_alloc, t_cycle = [], []
        for i in range(a.reps + 1):
            r = eng.allocate()
            util.assert_same_decisions(ref.decisions, r.decisions, f"W={W} allocate")
            res, gev, gorder, _ = eng.cycle(FULL_LIST)
            util.assert_same_decisions(e.decisions, res.decisions, f"W={W} cycle")
            assert (gev == eev).all() and (gorder == eorder).all()
            if i:                                                      # the first round is the warm-up
                t_alloc.append(r.stats.gpu_ms)
                t_cycle.append(res.stats.gpu_ms)
        row = {"W": W, "allocate_ms": float(np.median(t_alloc)), "cycle_ms": float(np.median(t_cycle)),
               "scans": int(r.stats.scans), "launches": int(r.stats.kernel_launches), "pipeline": int(r.stats.pipeline), "evictions": int(gev.sum())}
        out["rows"].append(row)
        print(json.dumps(row), flush=True)
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
