"""What InterPodAffinityPriority costs a preempt sweep on the GPU: a cluster of C3's size (50000 pending tasks, 5000 PodGroups, 5000
nodes) in three oversubscribed queues with soft hostname anti-affinity on every PodGroup (synth.add_pod_pref), kb_preempt from the
loaded state, podaffinity.weight 1 (passes 2-4 before every sweep, the score in it) against
podaffinity.weight 0 (the priority weighs nothing: the sweep alone).  Prints the GPU time per executed sweep of both and the difference.
    python tools/evict_pass_cost.py [preemptable_frac] [reps]"""
import copy, json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kube_batch_b200 import engine, synth

frac = float(sys.argv[1]) if len(sys.argv) > 1 else 0.4
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
snap = synth.add_pod_pref(synth.random_session(3, tasks=50000, jobs=5000, nodes=5000, queues=3, oversub=2.0), 1.0)
conf = synth.config_conf("c3")
run = synth.running_of(snap, frac)
try:
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as ex:                      # the card is named beside the numbers when nvidia-smi is there
    gpu = f"unknown ({ex})"
out = {"workload": f"{snap.T} pending tasks / {snap.N} nodes, every PodGroup with soft hostname anti-affinity "
                   f"({len(snap.meta['pod_pref_kinds'])} pod kinds), kb_preempt from the loaded state", "gpu": gpu}
eng = engine.Engine(0)
for w in ("1", "0"):
    c = copy.deepcopy(conf)
    for tier in c.tiers:
        for opt in tier:
            if opt.name == "nodeorder":
                opt.arguments = dict(opt.arguments, **{"podaffinity.weight": w})
    eng.load(snap, c).load_running(run)
    eng.preempt()                                # warm-up
    rows = []
    for _ in range(reps):
        res, ev, order = eng.preempt()
        st = res.stats
        rows.append((st.gpu_ms, int(st.evict_sweeps), int(st.evictions)))
    ms = sorted(r[0] for r in rows)
    sweeps = rows[0][1]
    out[f"podaffinity.weight {w}"] = {"gpu_ms_min": ms[0], "gpu_ms_median": ms[len(ms) // 2], "sweeps": sweeps, "evictions": rows[0][2],
                                      "us_per_sweep_median": 1e3 * ms[len(ms) // 2] / max(1, sweeps)}
eng.close()
a, b = out["podaffinity.weight 1"], out["podaffinity.weight 0"]
out["pass_cost_us_per_sweep"] = a["us_per_sweep_median"] - b["us_per_sweep_median"]
print(json.dumps(out, indent=1))
