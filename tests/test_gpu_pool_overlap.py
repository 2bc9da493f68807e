"""`-m gpu`: the pool builder of the persistent pipeline (kb_pipe.cuh, pipe_build) builds the next visit chain's candidate pool
while the main warp finishes the current chain.  The pool is taken when the visit has the predicted class (hit) and thrown away
at the visit start otherwise (miss: minMember below the job size lets jobs yield and re-enter the queue out of the static order), and
dropped without a wait when the chain goes on with another run of its class (cancelled).  Sessions with several queues, where the
queue heap reorders the visits, do not build ahead.  Every path must give the oracle's decisions bit for bit; the timing-mode
counters show that the hit and the miss path were taken."""
import os

import pytest

from kube_batch_b200 import engine, synth
from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def timed_eng():
    old = os.environ.get("KB_PIPE_TIMING")
    os.environ["KB_PIPE_TIMING"] = "1"          # read at engine creation: the build counters are kept in timing mode only
    try:
        e = engine.Engine(device=0)
    finally:
        if old is None:
            del os.environ["KB_PIPE_TIMING"]
        else:
            os.environ["KB_PIPE_TIMING"] = old
    yield e
    e.close()


def _check(eng, snap, conf, what):
    o = kbo.allocate(snap, conf)
    eng.load(snap, conf)
    r = eng.allocate()
    util.assert_same_decisions(o.decisions, r.decisions, what)
    util.assert_same_state(o, eng.node_state(), eng.order_state(), what)
    assert r.stats.pipeline == 1, f"{what}: the session did not run on cycle_kernel"
    return r.stats


def test_pool_builds_hit_and_miss_against_the_oracle(timed_eng):
    used = missed = 0
    conf = PluginConf.default()
    sessions = [("c2", synth.make("c2")[0])]
    for seed in range(6):
        sessions.append((f"seed{seed}", synth.random_session(seed, tasks=1500, jobs=150, nodes=300, queues=1 + (seed == 5),
                                                            min_member_frac=(0.0, 0.5, 1.0)[seed % 3], oversub=1.3)))
    for what, snap in sessions:
        st = _check(timed_eng, snap, conf, what)
        used += st.pipe_builds_used
        missed += st.pipe_builds_missed
    assert used > 0, "no pool built ahead was ever taken"
    assert missed > 0, "no pool built ahead was ever thrown away at a visit start"


@pytest.mark.parametrize("seed,frac", [(101, 0.0), (102, 0.5), (103, 1.0)])
def test_pool_builder_without_timing_mode(seed, frac):
    eng = engine.Engine(device=0)
    try:
        snap = synth.random_session(seed, tasks=2000, jobs=200, nodes=400, queues=1, min_member_frac=frac)
        _check(eng, snap, PluginConf.default(), f"seed{seed}/f{frac}")
    finally:
        eng.close()
