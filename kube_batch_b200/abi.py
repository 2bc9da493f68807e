"""ctypes mirror of include/kbgpu.h (the C ABI of libkbgpu.so).

Field order and types must match the header exactly; tests/test_abi.py cross-checks the struct
sizes against a C program compiled from the header.
"""
from __future__ import annotations

import ctypes as C

KB_ENGINE_NO_OVERLAP = 1 << 0
KB_ENGINE_FORCE_OVERLAP = 1 << 1
KB_ENGINE_CHAIN_OFF = 1 << 2
KB_ENGINE_CHAIN2 = 1 << 3
KB_ENGINE_CHAIN4 = 1 << 4
KB_ENGINE_NO_PIPE = 1 << 5
KB_ENGINE_SHARD = 1 << 6
KB_ABI_VERSION = 3
KB_MAX_R = 32
KB_MAX_W = 16
# kb_core.h: sessions above either narrow capacity run the wide (R) or wide-atom (W) kernel instances, never both
KB_NARROW_R = 8
KB_NARROW_W = 4
KB_MAX_AFF_TERMS = 4
KB_MAX_PREF_TERMS = 4
KB_MAX_Q = 65536

KB_OK = 0
KB_E_BADARG = -1
KB_E_UNSUPPORTED_PLUGIN = -2
KB_E_CUDA = -3
KB_E_NCCL = -4
KB_E_STATE = -5
KB_E_UNSUPPORTED_FEATURE = -6

KB_NODE_NOT_READY = 1 << 0
KB_NODE_NET_UNAVAILABLE = 1 << 1
KB_NODE_UNSCHEDULABLE = 1 << 2
KB_NODE_MEM_PRESSURE = 1 << 3
KB_NODE_DISK_PRESSURE = 1 << 4
KB_NODE_PID_PRESSURE = 1 << 5

KB_TASK_BEST_EFFORT_QOS = 1 << 0
KB_TASK_HAS_POD_AFFINITY = 1 << 1
KB_SNAPSHOT_PLACED_POD_AFFINITY = 1 << 0
KB_SNAPSHOT_LISTED_POD_WITHOUT_NODE = 1 << 1
KB_TASK_HAS_PREFERRED_NODE_AFFINITY = 1 << 2
KB_TASK_AFF_SELF_MATCH = 1 << 3
KB_MAX_AFF_GROUPS = 4096
KB_XGROUP_FORBID = 1
KB_XGROUP_CONTRIB = 2

KB_KIND_NONE = 0
KB_KIND_ALLOCATED = 1
KB_KIND_PIPELINED = 2
KB_KIND_SKIPPED = 3

_pd = C.POINTER(C.c_double)
_pu32 = C.POINTER(C.c_uint32)
_pi32 = C.POINTER(C.c_int32)
_pi64 = C.POINTER(C.c_int64)
_pu64 = C.POINTER(C.c_uint64)

# (field name, ctypes pointer type, numpy dtype, shape expression in terms of R W N T J Q A)
SNAPSHOT_ARRAYS = [
    ("node_idle", _pd, "f8", "RN"),
    ("node_releasing", _pd, "f8", "RN"),
    ("node_used", _pd, "f8", "RN"),
    ("node_allocatable", _pd, "f8", "RN"),
    ("node_alloc_present", _pu32, "u4", "N"),
    ("node_alloc_cpu", _pi64, "i8", "N"),
    ("node_alloc_mem", _pi64, "i8", "N"),
    ("node_nz_cpu", _pi64, "i8", "N"),
    ("node_nz_mem", _pi64, "i8", "N"),
    ("node_pods", _pi32, "i4", "N"),
    ("node_max_pods", _pi32, "i4", "N"),
    ("node_flags", _pu32, "u4", "N"),
    ("node_labels", _pu64, "u8", "WN"),
    ("node_taints", _pu64, "u8", "WN"),
    ("node_ports", _pu64, "u8", "WN"),
    ("task_initreq", _pd, "f8", "RT"),
    ("task_resreq", _pd, "f8", "RT"),
    ("task_res_present", _pu32, "u4", "T"),
    ("task_nz_cpu", _pi64, "i8", "T"),
    ("task_nz_mem", _pi64, "i8", "T"),
    ("task_sel_req", _pu64, "u8", "WT"),
    ("task_aff_terms", _pu64, "u8", "AWT"),
    ("task_n_aff_terms", _pu32, "u4", "T"),
    ("task_tol", _pu64, "u8", "WT"),
    ("task_port_own", _pu64, "u8", "WT"),
    ("task_port_conflict", _pu64, "u8", "WT"),
    ("task_flags", _pu32, "u4", "T"),
    ("task_prio", _pi32, "i4", "T"),
    ("task_ctime", _pi64, "i8", "T"),
    ("task_uid_rank", _pu32, "u4", "T"),
    ("job_task_off", _pu32, "u4", "J1"),
    ("job_min_avail", _pi32, "i4", "J"),
    ("job_ready0", _pi32, "i4", "J"),
    ("job_alloc0", _pd, "f8", "RJ"),
    ("job_alloc0_present", _pu32, "u4", "J"),
    ("job_queue", _pu32, "u4", "J"),
    ("job_prio", _pi32, "i4", "J"),
    ("job_ctime", _pi64, "i8", "J"),
    ("queue_weight", _pi32, "i4", "Q"),
    ("queue_ctime", _pi64, "i8", "Q"),
    ("task_n_pref_terms", _pu32, "u4", "T"),
    ("task_pref_terms", _pu64, "u8", "PWT"),
    ("task_pref_weights", _pi32, "i4", "PT"),
]


# kb_pod_affinity arrays: (field, ctypes element type, numpy dtype)
POD_AFFINITY_ARRAYS = [
    ("node_domain", C.c_int32, "i4"),
    ("keyset_domains", C.c_uint32, "u4"),
    ("group_keyset", C.c_uint32, "u4"),
    ("group_count0", C.c_int32, "i4"),
    ("group_total0", C.c_int32, "i4"),
    ("task_forbid", C.c_uint64, "u8"),
    ("task_need", C.c_int32, "i4"),
    ("task_contrib", C.c_uint64, "u8"),
    ("task_kind", C.c_int32, "i4"),
    ("node_kind_count0", C.c_int32, "i4"),
    ("kind_unbound", C.c_uint8, "u1"),
    ("task_weight_off", C.c_uint32, "u4"),
    ("weight_kind", C.c_int32, "i4"),
    ("weight_keyset", C.c_int32, "i4"),
    ("weight_value", C.c_int64, "i8"),
]
# groups >= 64 (include/kbgpu.h): optional, NULL when the dict has no such key (sessions with at most 64 groups)
POD_AFFINITY_XARRAYS = [
    ("task_xgroup_off", C.c_uint32, "u4"),
    ("task_xgroup", C.c_uint32, "u4"),
]


class kb_pod_affinity(C.Structure):
    """include/kbgpu.h kb_pod_affinity: inter-pod (anti)affinity, flattened by builder.py."""
    _fields_ = [
        ("n_keysets", C.c_uint32),
        ("n_groups", C.c_uint32),
        ("n_kinds", C.c_uint32),
        ("n_weights", C.c_uint32),
        ("first_unbound_node", C.c_int32),
        ("reserved", C.c_uint32),
    ] + [(name, C.POINTER(ct)) for name, ct, _ in POD_AFFINITY_ARRAYS + POD_AFFINITY_XARRAYS]


def pod_affinity_to_c(pa):
    """dict (builder.py) -> (kb_pod_affinity, keep-alive list)."""
    import numpy as np
    r = kb_pod_affinity()
    r.n_keysets = int(pa["n_keysets"]); r.n_groups = int(pa["n_groups"]); r.n_kinds = int(pa["n_kinds"])
    r.n_weights = int(pa["n_weights"]); r.first_unbound_node = int(pa["first_unbound_node"])
    keep = []
    for name, ct, dt in POD_AFFINITY_ARRAYS:
        a = np.ascontiguousarray(pa[name], dtype=np.dtype(dt)).reshape(-1)
        if a.size == 0:
            a = np.zeros(1, dtype=np.dtype(dt))
        keep.append(a)
        setattr(r, name, a.ctypes.data_as(C.POINTER(ct)))
    for name, ct, dt in POD_AFFINITY_XARRAYS:
        if pa.get(name) is None:
            continue
        a = np.ascontiguousarray(pa[name], dtype=np.dtype(dt)).reshape(-1)
        if a.size == 0:
            a = np.zeros(1, dtype=np.dtype(dt))
        keep.append(a)
        setattr(r, name, a.ctypes.data_as(C.POINTER(ct)))
    return r, keep


class kb_snapshot(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32),
        ("R", C.c_uint32),
        ("W", C.c_uint32),
        ("N", C.c_uint32),
        ("T", C.c_uint32),
        ("J", C.c_uint32),
        ("Q", C.c_uint32),
        ("flags", C.c_uint32),
    ] + [(name, ptr) for name, ptr, _, _ in SNAPSHOT_ARRAYS] + [("pod_affinity", C.POINTER(kb_pod_affinity))]


class kb_plugin_option(C.Structure):
    _fields_ = [
        ("name", C.c_char_p),
        ("enabled_job_order", C.c_uint8),
        ("enabled_job_ready", C.c_uint8),
        ("enabled_job_pipelined", C.c_uint8),
        ("enabled_task_order", C.c_uint8),
        ("enabled_preemptable", C.c_uint8),
        ("enabled_reclaimable", C.c_uint8),
        ("enabled_queue_order", C.c_uint8),
        ("enabled_predicate", C.c_uint8),
        ("enabled_node_order", C.c_uint8),
        ("n_args", C.c_uint32),
        ("arg_keys", C.POINTER(C.c_char_p)),
        ("arg_values", C.POINTER(C.c_char_p)),
    ]


class kb_tier(C.Structure):
    _fields_ = [("n_plugins", C.c_uint32), ("plugins", C.POINTER(kb_plugin_option))]


class kb_plugin_conf(C.Structure):
    _fields_ = [("n_tiers", C.c_uint32), ("tiers", C.POINTER(kb_tier))]


class kb_engine_opts(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32),
        ("device", C.c_int32),
        ("rank", C.c_int32),
        ("world_size", C.c_int32),
        ("nccl_unique_id", C.c_void_p),
        ("flags", C.c_uint32),
    ]


class kb_decision(C.Structure):
    _fields_ = [
        ("node", C.c_int32),
        ("kind", C.c_uint8),
        ("dispatched", C.c_uint8),
        ("reserved", C.c_uint16),
        ("step", C.c_uint32),
        ("dispatch_step", C.c_uint32),
    ]


class kb_stats(C.Structure):
    _fields_ = [
        ("pairs_logical", C.c_uint64),
        ("pairs_scanned", C.c_uint64),
        ("pairs_replayed", C.c_uint64),
        ("tasks_processed", C.c_uint32),
        ("tasks_allocated", C.c_uint32),
        ("tasks_pipelined", C.c_uint32),
        ("jobs_ready", C.c_uint32),
        ("visits", C.c_uint32),
        ("kernel_launches", C.c_uint32),
        ("n_classes", C.c_uint32),
        ("gpu_ms", C.c_float),
        ("load_ms", C.c_float),
        ("h2d_bytes", C.c_uint64),
        ("d2h_bytes", C.c_uint64),
        ("scans", C.c_uint32),
        ("rescans", C.c_uint32),
        ("cyc_scan", C.c_uint64),
        ("cyc_merge", C.c_uint64),
        ("cyc_replay", C.c_uint64),
        ("cyc_total", C.c_uint64),
        ("cyc_steps", C.c_uint64),
        ("cyc_ctl", C.c_uint64),
        ("predictions", C.c_uint32),
        ("mispredictions", C.c_uint32),
        ("exchange_mode", C.c_uint32),
        ("chain_hits", C.c_uint32),
        ("pipeline", C.c_uint32),
        ("pipe_requests", C.c_uint32),
        ("pipe_urgent", C.c_uint32),
        ("pipe_extends", C.c_uint32),
        ("pipe_patched", C.c_uint32),
        ("pipe_patch_entries", C.c_uint32),
        ("evictions", C.c_uint32),
        ("evict_sweeps", C.c_uint32),
        ("cyc_ring", C.c_uint64),
        ("cyc_plan", C.c_uint64),
        ("pipe_builds_used", C.c_uint32),
        ("pipe_builds_missed", C.c_uint32),
        ("pipe_builds_cancelled", C.c_uint32),
    ]


KB_RUNNING_CRITICAL = 1 << 0
KB_RUNNING_AFF_MEMBER = 1 << 1


class kb_running(C.Structure):
    """Running tasks one by one (include/kbgpu.h kb_running): what reclaim / preempt walk."""
    _fields_ = [
        ("n", C.c_uint32),
        ("reserved0", C.c_uint32),
        ("node", C.POINTER(C.c_uint32)),
        ("job", C.POINTER(C.c_uint32)),
        ("resreq", C.POINTER(C.c_double)),
        ("res_present", C.POINTER(C.c_uint32)),
        ("prio", C.POINTER(C.c_int32)),
        ("ctime", C.POINTER(C.c_int64)),
        ("uid_rank", C.POINTER(C.c_uint32)),
        ("flags", C.POINTER(C.c_uint32)),
        ("job_waiting0", C.POINTER(C.c_int32)),
        ("aff_group_off", C.POINTER(C.c_uint32)),
        ("aff_group", C.POINTER(C.c_uint32)),
    ]


def running_to_c(running, R: int, J: int = 0):
    """dict of arrays (builder.py meta["running"]) -> (kb_running, keep-alive list)."""
    import numpy as np
    n = 0 if running is None else len(running["node"])
    spec = (("node", np.uint32), ("job", np.uint32), ("resreq", np.float64), ("res_present", np.uint32), ("prio", np.int32),
            ("ctime", np.int64), ("uid_rank", np.uint32), ("flags", np.uint32))
    arrs = {}
    for k, dt in spec:
        a = np.ascontiguousarray(running[k], dtype=dt) if n else np.zeros((R, 1) if k == "resreq" else 1, dtype=dt)
        arrs[k] = a
    if n:
        assert arrs["resreq"].shape == (R, n)
    r = kb_running()
    r.n = n
    ctypes_of = {np.uint32: C.c_uint32, np.float64: C.c_double, np.int32: C.c_int32, np.int64: C.c_int64}
    for k, dt in spec:
        setattr(r, k, arrs[k].ctypes.data_as(C.POINTER(ctypes_of[dt])))
    keep = list(arrs.values())
    jw = None if running is None else running.get("job_waiting0")
    if jw is not None:
        jw = np.ascontiguousarray(jw, dtype=np.int32)
        r.job_waiting0 = jw.ctypes.data_as(C.POINTER(C.c_int32))
        keep.append(jw)
    # the counter groups of every Running task (builder.py meta["running_aff_groups"], merged in by the caller); NULL when absent
    for k in ("aff_group_off", "aff_group"):
        a = None if running is None else running.get(k)
        if a is None:
            continue
        a = np.ascontiguousarray(a, dtype=np.uint32).reshape(-1)
        if a.size == 0:
            a = np.zeros(1, dtype=np.uint32)
        setattr(r, k, a.ctypes.data_as(C.POINTER(C.c_uint32)))
        keep.append(a)
    return r, keep


DECISION_DTYPE = [
    ("node", "<i4"),
    ("kind", "u1"),
    ("dispatched", "u1"),
    ("reserved", "<u2"),
    ("step", "<u4"),
    ("dispatch_step", "<u4"),
]
