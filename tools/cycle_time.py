"""Time kb_cycle (the shipped action list on ONE session) on a BASELINE config + its Running filler pods, and check it against
the oracle.   python tools/cycle_time.py c3 [preemptable_frac] [oracle:0|1] [node_pref_frac]
node_pref_frac > 0: that share of the PodGroups carries preferred zone affinity (synth.add_node_pref)."""
import sys, os, time, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from kube_batch_b200 import engine, synth, digest

name = sys.argv[1] if len(sys.argv) > 1 else "c3"
frac = float(sys.argv[2]) if len(sys.argv) > 2 else 0.3
with_oracle = int(sys.argv[3]) if len(sys.argv) > 3 else 1
pref_frac = float(sys.argv[4]) if len(sys.argv) > 4 else 0.0
acts = ("reclaim", "allocate", "backfill", "preempt")
snap, conf = synth.make(name)
if pref_frac > 0:
    synth.add_node_pref(snap, pref_frac)
run = synth.running_of(snap, frac)
eng = engine.Engine(0)
t0 = time.time(); eng.load(snap, conf).load_running(run); t1 = time.time()
workload = f"{name}: {snap.T} pending tasks / {snap.N} nodes / {len(run['node'])} Running pods one by one, {frac:.0%} of the filler PodGroups preemptable"
if pref_frac > 0:
    workload += f", {pref_frac:.0%} of the PodGroups with preferred zone affinity ({snap.meta['pref_tasks']} tasks)"
out = {"workload": workload, "actions": list(acts), "load_ms": 1e3 * (t1 - t0)}
for rep in range(3):
    t0 = time.time(); res, ev, order, bounds = eng.cycle(acts); t1 = time.time()
    st = res.stats
    out[f"rep{rep}"] = {"wall_ms": 1e3 * (t1 - t0), "gpu_ms": st.gpu_ms, "evictions": int(st.evictions), "evict_sweeps": int(st.evict_sweeps),
                        "preemptor_tasks+allocate_tasks": int(st.tasks_processed), "allocated": int((res.decisions["kind"] == 1).sum()),
                        "pipelined": int((res.decisions["kind"] == 2).sum()), "launches": int(st.kernel_launches),
                        "bounds[step,evictions] per action": bounds.tolist()}
if with_oracle:
    from oracle import kbo
    t0 = time.time(); o, oev, oorder = kbo.cycle(snap, conf, actions=acts, running=run, threads=16); t1 = time.time()
    same = bool((o.decisions == res.decisions).all() and (oev == ev).all() and (oorder == order).all())
    out["oracle"] = {"seconds": t1 - t0, "threads": 16, "evictions": int(oev.sum()), "bit_exact": same}
print(json.dumps(out, indent=1))
if with_oracle and not out["oracle"]["bit_exact"]:
    sys.exit(1)
