"""reclaim / preempt with preferred inter-pod (anti)affinity on the GPU (kb_evict_kernels.cu: passes 2-4 for InterPodAffinityPriority's
weights per domain and min / max count, then the sweep; the master thread keeps kind_count / first_unbound through Pipeline and
Statement discard) through the C ABI.  The hand vectors and random clusters of test_evict_pod_pref run here with every outcome also
checked on the GPU against the oracle (and the emulation, which checks itself against the oracle); a C3-sized cluster with soft
spread on 15 % of its PodGroups runs against the emulation."""
from __future__ import annotations

import time

import pytest

from kube_batch_b200 import abi, synth
from kube_batch_b200.snapshot import PluginConf
import util
import test_evict_pod_pref as tp
from test_evict_parity import compare

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from kube_batch_b200 import engine
    e = engine.Engine(0)
    yield e
    e.close()


def _run(eng, acts):
    if len(acts) == 1 and acts[0] in ("reclaim", "preempt"):
        return eng.reclaim() if acts[0] == "reclaim" else eng.preempt()
    res, gev, gorder, _ = eng.cycle(acts)
    return res, gev, gorder


@pytest.fixture
def on_gpu(eng, monkeypatch):
    """test_evict_pod_pref.run_both, plus the same session through the C ABI on the GPU"""
    cpu = tp.run_both

    def both(s, tiers, acts, what):
        o, ev, order = cpu(s, tiers, acts, what)
        eng.load(s, tiers).load_running(s.meta["running"])
        res, gev, gorder = _run(eng, acts)
        compare(f"gpu {what}", o, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
        util.assert_same_decisions(o.decisions, res.decisions, f"gpu {what}")
        return o, ev, order

    monkeypatch.setattr(tp, "run_both", both)
    return tp


VECTOR_TESTS = sorted(n for n in dir(tp) if n.startswith("test_") and n[5].isdigit())


@pytest.mark.parametrize("name", VECTOR_TESTS)
def test_hand_vectors_on_the_gpu(on_gpu, name):
    getattr(on_gpu, name)()


@pytest.mark.parametrize("seed", [0, 1, 2, 3, 5, 8, 13, 21])
def test_random_clusters_on_the_gpu(on_gpu, seed):
    on_gpu.test_random_clusters_on_the_emulation(seed)


def test_members_of_unread_groups_on_the_gpu(on_gpu):
    on_gpu.test_members_of_unread_groups_are_evicted_without_withholding()


def test_a_class_that_reads_a_group_is_still_refused_on_the_gpu(eng):
    """14 of its 28 pending tasks carry forbid bits: kb_session_load_running refuses it with the message it always had"""
    from kube_batch_b200.engine import KbError
    s = tp.aff_gen.random_affinity_session(77, n_nodes=20, n_groups=10).flatten()
    eng.load(s, PluginConf.default())
    with pytest.raises(KbError) as ex:
        eng.load_running(s.meta["running"])
    assert ex.value.code == abi.KB_E_UNSUPPORTED_FEATURE
    assert "reclaim / preempt in this session with inter-pod affinity are outside this build" in str(ex.value)


def test_c3_sized_cluster_with_soft_spread(eng):
    """C3's size (50000 pending tasks, 5000 PodGroups, 5000 nodes) in three oversubscribed queues, 15 % of the PodGroups with soft
    hostname anti-affinity (synth.add_pod_pref), 40 % of the filler PodGroups preemptable: the shipped action list on the counter
    path, GPU vs the emulation, bit-exact."""
    s = synth.add_pod_pref(synth.random_session(3, tasks=50000, jobs=5000, nodes=5000, queues=3, oversub=2.0), 0.15)
    conf = synth.config_conf("c3")
    run = synth.running_of(s, 0.4)
    acts = ("reclaim", "allocate", "backfill", "preempt")
    t0 = time.time()
    g, ev, order = util.emu_cycle(s, conf, acts, run, mode=1)
    t_emu = time.time() - t0
    eng.load(s, conf).load_running(run)
    for rep in range(2):
        res, gev, gorder, _ = eng.cycle(acts)
        compare(f"c3-sized soft spread rep {rep}", g, ev, order, res, gev, gorder, (eng.node_state(), eng.order_state()))
        util.assert_same_decisions(g.decisions, res.decisions, f"c3-sized soft spread rep {rep}")
    st = res.stats
    soft = s.pod_affinity["task_kind"][:s.T] >= 0
    print(f"\nc3-sized cluster, {int(soft.sum())} soft-spread tasks, {len(s.meta['pod_pref_kinds'])} pod kinds: path visit_kernel<0,1> "
          f"(counters) + evict_kernel passes 2-4, launches {int(st.kernel_launches)}, gpu_ms {st.gpu_ms:.2f}, evictions "
          f"{int(st.evictions)}, evict sweeps {int(st.evict_sweeps)}, pipelined {int((res.decisions['kind'] == abi.KB_KIND_PIPELINED).sum())} "
          f"(soft spread {int(((res.decisions['kind'] == abi.KB_KIND_PIPELINED) & soft).sum())}); emulation {t_emu:.1f} s")
    assert int(st.evictions) > 0 and ((res.decisions["kind"] == abi.KB_KIND_PIPELINED) & soft).any()
