"""reclaim / preempt evicting members of host-level anti-affinity groups on the GPU (kb_evict_kernels.cu: the master thread updates the
member counts and bits of the node records between two sweeps; evict_scan_kernel folds the Allocated members of the cycle into the
counts).  Through the C ABI against the CPU emulation of the same algorithm and against the status-following oracle
(tests/follow_oracle.py), bit-exact."""
from __future__ import annotations

import numpy as np
import pytest

from kube_batch_b200 import abi, synth
from oracle import kbo
import aff_gen
import aff_gen_many
import follow_oracle
import util
from test_evict_parity import compare, tier_variants
from test_evict_aff_members import LISTS, VECTORS, placements, tiers, with_lists

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from kube_batch_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()


def _run(eng, acts):
    if len(acts) == 1:
        return eng.reclaim() if acts[0] == "reclaim" else eng.preempt()
    res, gev, gorder, _ = eng.cycle(acts)
    return res, gev, gorder


def _gpu_vs_emu(eng, s, tr, acts, run, what):
    eng.load(s, tr).load_running(run)
    res, gev, gorder = _run(eng, acts)
    g, ev, order = util.emu_cycle(s, tr, acts, run, mode=1)
    compare(what, g, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
    util.assert_same_decisions(g.decisions, res.decisions, what)
    return res, gev, gorder


@pytest.mark.parametrize("case", VECTORS, ids=lambda c: c[0].split(":")[0])
def test_hand_vectors_on_the_gpu(eng, case):
    name, make, acts, want, want_ev, _ = case
    s = make()
    res, gev, gorder = _gpu_vs_emu(eng, s, tiers(), acts, with_lists(s), name)
    assert placements(s, res) == want, name


def _clusters():
    for seed in (0, 1, 2, 3, 5, 8, 13):
        yield f"seed {seed}", aff_gen.evict_spread_cluster(seed, members_running=True)
    for seed in (0, 1):
        yield f"many seed {seed}", aff_gen_many.evict_spread_cluster(seed, members_running=True, n_apps=300, n_pod_groups=90, W=2)


@pytest.mark.parametrize("case", range(9))
def test_random_clusters_on_the_gpu(eng, case):
    what, s = list(_clusters())[case]
    if s.pod_affinity is None:
        pytest.skip("no PodGroup drew the spread")
    for tname, tr in tier_variants():
        for acts in LISTS:
            res, gev, gorder = _gpu_vs_emu(eng, s, tr, acts, with_lists(s), f"{what} {tname} {acts}")
            o, ev, order = follow_oracle.cycle(s, tr, acts, with_lists(s))
            compare(f"{what} {tname} {acts} vs the oracle", o, ev, order, res, gev, gorder)


def member_cluster():
    """C3's size (50000 pending tasks, 5000 PodGroups, 5000 nodes) in three oversubscribed queues, so that reclaim and preempt evict,
    10 % of the PodGroups spread one per host and 10 % of the Running pods replicas of those Deployments"""
    s = synth.random_session(3, tasks=50000, jobs=5000, nodes=5000, queues=3, oversub=2.0)
    synth.add_host_spread(s, 0.1)
    run = synth.running_of(s, 0.4)
    lists = synth.add_running_members(s, run, 0.1)
    return s, synth.config_conf("c3"), run, lists


def test_c3_sized_cluster_with_members_evicted(eng):
    """the shipped action list: without the group lists the cycle is withheld (a member is evicted), with them the GPU returns the
    emulation's result"""
    s, conf, run, lists = member_cluster()
    acts = ("reclaim", "allocate", "backfill", "preempt")
    member = (run["flags"] & abi.KB_RUNNING_AFF_MEMBER) != 0
    from kube_batch_b200.engine import KbError
    eng.load(s, conf).load_running(run)
    with pytest.raises(KbError) as ex:
        eng.cycle(acts)
    assert ex.value.code == abi.KB_E_UNSUPPORTED_FEATURE and "evicted" in str(ex.value)
    res, gev, gorder = _gpu_vs_emu(eng, s, conf, acts, dict(run, **lists), "c3-sized members")
    assert (gev & member).any()
    res, gev, gorder, _ = eng.cycle(acts)
    st = res.stats
    print(f"\nc3-sized cluster, {int(member.sum())} Running members: gpu_ms {st.gpu_ms:.2f} launches {int(st.kernel_launches)} "
          f"evictions {int(st.evictions)} (members {int((gev & member).sum())})")
