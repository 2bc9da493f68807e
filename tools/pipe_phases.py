"""Phase split of the persistent pipeline's main warp per visit chain, and the hit rate of the pool builder.

    python tools/pipe_phases.py [config ...]        (default: c3 c4; runs with KB_PIPE_TIMING=1)

Cycles per visit chain (clock64 of the main warp):
  list wait  = waiting for the prepared list of a visit built on the main warp
  pool build = visit start to the first step, minus the list wait (on a hit: waiting for the builder's pool)
  step loop  = the runs' step loops
  post-loop  = decisions, sums, shares and control plane after the step loops, plus the chain's hot-ring / write-back stage
builds used / missed / cancelled: pools of the next chain built ahead and taken / not fitting the visit / dropped because the
chain went on."""
import os
import sys

os.environ["KB_PIPE_TIMING"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from kube_batch_b200 import engine, synth  # noqa: E402

eng = engine.Engine(0)
for name in sys.argv[1:] or ["c3", "c4"]:
    snap, conf = synth.make(name)
    eng.load(snap, conf)
    eng.allocate()                      # warm-up
    s = eng.allocate().stats
    n = max(1, s.scans)
    wait, build = s.cyc_total / n, (s.cyc_scan - s.cyc_total) / n
    loop, post = s.cyc_merge / n, (s.cyc_steps - s.cyc_merge + s.cyc_ctl + s.cyc_ring) / n
    b = s.pipe_builds_used + s.pipe_builds_missed + s.pipe_builds_cancelled
    print(f"{name}: {s.gpu_ms:.2f} ms, {s.scans} visit chains, {1e3 * s.gpu_ms / n:.2f} us per chain; cycles per chain: "
          f"list wait {wait:.0f}, pool build {build:.0f}, step loop {loop:.0f}, post-loop {post:.0f}; "
          f"builds used {s.pipe_builds_used}, missed {s.pipe_builds_missed}, cancelled {s.pipe_builds_cancelled} "
          f"(hit rate {s.pipe_builds_used / max(1, b):.1%})")
eng.close()
