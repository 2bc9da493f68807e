"""CPU parity on boundary-state sessions (tests/edge_gen.py): epsilon fits, pod caps reached partway through a run, Allocate ->
Pipeline flips, zero and irregular capacities, 10 / 11 milli scalar requests, runs of more than 40 placements on one node.  The
emulation (every launch mode), backfill and the full action list against the oracle; each test also asserts, from the oracle's
own decisions and final state, that the sessions reached the edges they were built for."""
import numpy as np
import pytest

from kube_batch_b200.snapshot import PluginConf
from oracle import kbo
import edge_gen as E
import util
from test_emu_parity import CONFS, check
from test_evict_parity import compare

EDGE_CONFS = ("default", "c2", "weights", "negweight", "nogang", "drf_first")
# (name, edge_session kwargs): R = 3 / W = 2 unless `wide`
VARIANTS = [("base", {}), ("multiqueue", {"queues": 3}), ("pref", {"pref": True}), ("wide", {"wide": True})]


def edge_confs():
    for cname in EDGE_CONFS:
        yield cname, CONFS[cname]
    yield "mostrequested", E.mostrequested_conf()


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("variant", [v[0] for v in VARIANTS])
def test_edge_sessions_emulation_against_the_oracle(variant, seed):
    kw = dict(VARIANTS)[variant]
    s = E.edge_session(100 * seed + len(variant), **kw)
    assert (s.R, s.W) == ((4, 3) if kw.get("wide") else (3, 2))
    # chained visits (modes 2 / 4) do not take classes with preferred terms: those run on the plain launches and the pipeline
    modes = (1, 5) if kw.get("pref") else (0, 1, 2, 4, 5)
    covs = []
    for cname, conf in edge_confs():
        for mode in modes:
            o, e = check(s, conf, f"edge {variant}/seed{seed}/{cname}/mode{mode}", mode=mode)
        covs.append(E.coverage(s, o))
    cov = E.merge(covs)
    print(f"edge {variant}/seed{seed}: N {s.N} T {s.T} coverage {cov}")
    E.assert_covered(cov, f"{variant}/seed{seed}")


@pytest.mark.parametrize("seed", range(3))
def test_edge_sessions_backfill(seed):
    s = E.edge_session(300 + seed, queues=1 + seed % 2, best_effort=True)
    covs = []
    for cname in ("default", "c2", "weights", "allocate_test"):
        for actions in (2, 3):
            o, e = check(s, CONFS[cname], f"edge backfill seed{seed}/{cname}/actions{actions}", actions=actions)
            if actions == 3:
                covs.append(E.coverage(s, o))
        check(s, CONFS[cname], f"edge backfill seed{seed}/{cname}/pipeline", actions=3, mode=5)
    cov = E.merge(covs)
    assert cov["nodes_at_pod_cap"] > 0 and cov["nodes_idle_cpu_in_epsilon"] > 0 and cov["zero_capacity_nodes_used"] > 0, cov


CYCLE = ("reclaim", "allocate", "backfill", "preempt")


@pytest.mark.parametrize("seed", range(4))
def test_edge_sessions_full_action_list(seed):
    """reclaim, allocate, backfill, preempt on one session, from the generator's Running pods (fillers of every node, terminating
    pods on the flip nodes) — the emulation against the oracle, evictions and final state included."""
    s = E.edge_session(500 + seed, queues=1 + seed % 3, best_effort=seed % 2 == 1, long_runs=seed < 2)
    run = s.meta["running"]
    assert len(run["node"]) > 20
    for cname, conf in (("default", PluginConf.default()), ("c2", CONFS["c2"]), ("weights", CONFS["weights"])):
        o, ev, order = kbo.cycle(s, conf, actions=CYCLE, running=run)
        g, gev, gorder = util.emu_cycle(s, conf, CYCLE, run)
        compare(f"edge cycle seed{seed}/{cname}", o, ev, order, g, gev, gorder, util.emu_states(g))
        assert (o.node_idle[0] > -10).all() and (o.node_idle[1] > -10 * 1024 * 1024).all()
