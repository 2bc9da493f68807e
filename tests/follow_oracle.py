"""The object-level oracle with util.PodLister following the Running tasks' status.

oracle/kb_oracle.cpp lists the pods of kbo_running as static `existing` pods (for_each_listed_pod): a Running pod that reclaim /
preempt evicts stays listed there.  The reference drops it: util.PodLister (plugins/util/util.go:37-85) only lists tasks whose status
is an AllocatedStatus (Bound, Binding, Running, Allocated), and an evicted task is Releasing — until a discarded Statement brings it
back to Running.  This module builds a variant of the same oracle source that knows which `existing` pod each kbo_running task is
and skips that pod while the task is not AllocatedStatus.  The source is rewritten at build time into a temporary directory (the
oracle itself stays as it is); every other line of the oracle is the same, and sessions in which no member of a counter group is
evicted give the same result as the oracle.  tests/test_evict_aff_members.py checks the engine's exact member bits against it."""
from __future__ import annotations

import ctypes as C
import fcntl
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import kbo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "oracle", "kb_oracle.cpp")

# (text in oracle/kb_oracle.cpp, replacement): each must occur exactly once
_EDITS = [
    ("thread_local std::shared_ptr<PodWorld> g_pod_world;",
     "thread_local std::shared_ptr<PodWorld> g_pod_world;\n"
     "// existing pod k -> the kbo_running task it is (-1: none), set by kbo_follow_set_running_pods before kbo_cycle\n"
     "thread_local std::vector<int32_t> g_run_of_existing;"),
    ("    for (const ExistingPod& e : pw->existing) if (e.listed) if (!fn(pw->pods[e.pod], (uint32_t)e.node)) return false;",
     "    for (size_t k = 0; k < pw->existing.size(); ++k) {\n"
     "      const ExistingPod& e = pw->existing[k];\n"
     "      if (!e.listed) continue;\n"
     "      if (k < g_run_of_existing.size() && g_run_of_existing[k] >= 0 &&\n"
     "          !AllocatedStatus(Tasks[(size_t)pw->T + (size_t)g_run_of_existing[k]].Status)) continue;   // evicted: Releasing\n"
     "      if (!fn(pw->pods[e.pod], (uint32_t)e.node)) return false;\n"
     "    }"),
    ('extern "C" {',
     'extern "C" {\n'
     "void kbo_follow_set_running_pods(const int32_t* run_of_existing, uint32_t n) {\n"
     "  g_run_of_existing.assign(run_of_existing, run_of_existing + n);\n"
     "}"),
]

_lib = None


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC).read()
        for old, new in _EDITS:
            assert src.count(old) == 1, f"oracle source changed: {old[:60]!r}"
            src = src.replace(old, new)
        tag = hashlib.sha1((src + open(os.path.join(ROOT, "include", "kbgpu.h")).read()).encode()).hexdigest()[:16]
        d = os.path.join(tempfile.gettempdir(), f"kbo_follow_{os.getuid()}_{tag}")
        os.makedirs(d, exist_ok=True)
        so = os.path.join(d, "libkbofollow.so")
        with open(os.path.join(d, ".lock"), "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if not os.path.exists(so):
                cpp = os.path.join(d, "kb_oracle_follow.cpp")
                open(cpp, "w").write(src)
                subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-pthread", "-shared",
                                       "-I", os.path.join(ROOT, "oracle"), "-I", os.path.join(ROOT, "include"),
                                       "-o", so + ".tmp", cpp])
                os.replace(so + ".tmp", so)
        L = C.CDLL(so)
        L.kbo_last_error.restype = C.c_char_p
        L.kbo_follow_set_running_pods.argtypes = [C.POINTER(C.c_int32), C.c_uint32]
        _lib = L
    return _lib


def running_of_existing(snap, running) -> np.ndarray:
    """existing pod k of snap.meta["pod_objects"] -> index of the kbo_running task it is, -1"""
    ex = snap.meta["pod_objects"]["existing"]
    idx = {name: i for i, name in enumerate(running["names"])}
    return np.array([idx.get(f"{p.namespace}/{p.name}", -1) for p in ex] or [-1], dtype=np.int32)


def cycle(snap, conf, actions, running):
    """kbo.cycle on the status-following variant -> (OracleOut, evicted, evict_order)"""
    L = lib()
    m = running_of_existing(snap, running) if snap.meta.get("pod_objects") is not None else np.full(1, -1, dtype=np.int32)
    L.kbo_follow_set_running_pods(m.ctypes.data_as(C.POINTER(C.c_int32)), C.c_uint32(len(m)))
    saved = kbo._lib
    kbo._lib = L
    try:
        return kbo.cycle(snap, conf, actions=actions, running=running)
    finally:
        kbo._lib = saved
        L.kbo_follow_set_running_pods(m.ctypes.data_as(C.POINTER(C.c_int32)), C.c_uint32(0))
