"""The shared arithmetic of kb_core.h / kb_aff.h against plain Python restatements of the reference (kube-batch, Go).

tests/probe/libkbprobe.so exposes every function twice: the KB_HD code compiled for the host (checked here, no GPU needed) and the
same code compiled for sm_90a (tests/test_gpu_core_arith.py, same cases, same references).  The device build of a function is
NOT the host build: div_0_to_10 estimates with MUFU.RCP instead of a float division, the double arithmetic goes through the
round-to-nearest intrinsics.  The references below are written from the Go source:
  Go int64 arithmetic   -> Python ints (`go_div` truncates towards zero like Go's `/`)
  Go float64 arithmetic -> Python floats (neither fuses a*b+c; int -> float conversions round to nearest)
The inputs sit where such code goes wrong: capacities that do not convert to float exactly, exact multiples and their neighbours,
fractions whose score lands within an ulp of an integer, the LessEqual epsilons, 32-bit score-field wrap-around."""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

_HERE = os.path.dirname(os.path.abspath(__file__))
_PROBE = os.path.join(_HERE, "probe", "libkbprobe.so")
MASK64 = (1 << 64) - 1
MIN_CPU, MIN_MEM, MIN_SCALAR = 10.0, 10.0 * 1024 * 1024, 10.0      # api/resource_info.go:68-70
_lib = None


def probe():
    global _lib
    if _lib is None:
        import fcntl
        with open(os.path.join(_HERE, "probe", ".build.lock"), "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            subprocess.check_call(["make", "-C", os.path.join(_HERE, "probe"), "-s"])
        L = C.CDLL(_PROBE)
        for f in ("kbp_div_0_to_10", "kbp_least_requested", "kbp_most_requested", "kbp_balanced", "kbp_le_func",
                  "kbp_res_less_equal", "kbp_aff_score", "kbp_add_pref_term", "kbp_aff_add_score", "kbp_eval_pair"):
            getattr(L, f).restype = C.c_int
        _lib = L
    return _lib


# ---------------------------------------------------------------- ctypes mirrors of kb::EvalConf / kb::ClassRec
KB_MAX_R, KB_MAX_W, KB_MAX_AFF_TERMS = 8, 4, 4


class EvalConf(C.Structure):
    _fields_ = [("R", C.c_uint32), ("W", C.c_uint32), ("predicates", C.c_uint32), ("mem_pressure", C.c_uint32),
                ("disk_pressure", C.c_uint32), ("pid_pressure", C.c_uint32), ("nodeorder", C.c_uint32), ("w_least", C.c_int32),
                ("w_most", C.c_int32), ("w_balanced", C.c_int32), ("score_bias", C.c_int64), ("fit_mode", C.c_uint32),
                ("pad0", C.c_uint32)]


class ClassRec(C.Structure):
    _fields_ = [("initreq", C.c_double * KB_MAX_R), ("resreq", C.c_double * KB_MAX_R), ("nz_cpu", C.c_int64), ("nz_mem", C.c_int64),
                ("sel_req", C.c_uint64 * KB_MAX_W), ("aff", (C.c_uint64 * KB_MAX_W) * KB_MAX_AFF_TERMS), ("tol", C.c_uint64 * KB_MAX_W),
                ("port_own", C.c_uint64 * KB_MAX_W), ("port_conflict", C.c_uint64 * KB_MAX_W), ("aff_own", C.c_uint64 * KB_MAX_W),
                ("n_aff", C.c_uint32), ("flags", C.c_uint32)]


# ---------------------------------------------------------------- entry points (device = 0: host build, 1: sm_90a build)
def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _i64(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.int64))


def _call(fn, device, n, *arrays):
    rc = fn(C.c_int(device), C.c_size_t(n), *[_ptr(a) if isinstance(a, np.ndarray) else a for a in arrays])
    assert rc == 0, f"{fn.__name__}: status {rc}"


def run_div(device, a, b):
    a, b = _i64(a), _i64(b)
    out = np.zeros(len(a), dtype=np.int64)
    _call(probe().kbp_div_0_to_10, device, len(a), a, b, out)
    return out


def run_requested(device, which, req, cap):
    req, cap = _i64(req), _i64(cap)
    out = np.zeros(len(req), dtype=np.int64)
    _call(getattr(probe(), f"kbp_{which}_requested"), device, len(req), req, cap, out)
    return out


def run_balanced(device, rc, cc, rm, cm):
    rc, cc, rm, cm = _i64(rc), _i64(cc), _i64(rm), _i64(cm)
    out = np.zeros(len(rc), dtype=np.int64)
    _call(probe().kbp_balanced, device, len(rc), rc, cc, rm, cm, out)
    return out


def run_le(device, l, r, diff):
    l, r, diff = (np.ascontiguousarray(np.asarray(x, dtype=np.float64)) for x in (l, r, diff))
    out = np.zeros(len(l), dtype=np.uint8)
    _call(probe().kbp_le_func, device, len(l), l, r, diff, out)
    return out.astype(bool)


def run_res_le(device, l, r):
    l, r = (np.ascontiguousarray(np.asarray(x, dtype=np.float64)) for x in (l, r))
    n, R = l.shape
    out = np.zeros(n, dtype=np.uint8)
    rc = probe().kbp_res_less_equal(C.c_int(device), C.c_size_t(n), C.c_int64(R), _ptr(l), _ptr(r), _ptr(out))
    assert rc == 0, rc
    return out.astype(bool)


def run_aff_score(device, count, mn, mx):
    count, mn, mx = _i64(count), _i64(mn), _i64(mx)
    out = np.zeros(len(count), dtype=np.int64)
    _call(probe().kbp_aff_score, device, len(count), count, mn, mx, out)
    return out


def run_add_pref_term(device, key, w, count, max_count):
    key = np.ascontiguousarray(np.asarray(key, dtype=np.uint64))
    w, count, max_count = _i64(w), _i64(count), _i64(max_count)
    out = np.zeros(len(key), dtype=np.uint64)
    _call(probe().kbp_add_pref_term, device, len(key), key, w, count, max_count, out)
    return out


def run_aff_add_score(device, key, w, score):
    key = np.ascontiguousarray(np.asarray(key, dtype=np.uint64))
    w, score = _i64(w), _i64(score)
    out = np.zeros(len(key), dtype=np.uint64)
    _call(probe().kbp_aff_add_score, device, len(key), key, w, score, out)
    return out


def run_eval_pair(device, geometry, cf: EvalConf, classes, tiles):
    n = len(classes)
    cls = (ClassRec * n)(*classes)
    key = np.zeros(n, dtype=np.uint64)
    fi = np.zeros(n, dtype=np.uint8)
    pok = np.zeros(n, dtype=np.uint8)
    rc = probe().kbp_eval_pair(C.c_int(device), C.c_int(geometry), C.c_size_t(n), C.byref(cf), C.cast(cls, C.c_void_p), _ptr(tiles),
                               _ptr(key), _ptr(fi), _ptr(pok))
    assert rc == 0, rc
    return key, fi.astype(bool), pok.astype(bool)


# ---------------------------------------------------------------- references (Go source -> Python)
def go_div(a: int, b: int) -> int:
    """Go's int64 `/`: truncates towards zero."""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def ref_least(req: int, cap: int) -> int:          # least_requested.go:49-58
    if cap == 0 or req > cap:
        return 0
    return go_div((cap - req) * 10, cap)


def ref_most(req: int, cap: int) -> int:           # most_requested.go:52-61
    if cap == 0 or req > cap:
        return 0
    return go_div(req * 10, cap)


def ref_balanced(rc: int, cc: int, rm: int, cm: int) -> int:    # balanced_resource_allocation.go:42-79
    cf = 1.0 if cc == 0 else float(rc) / float(cc)
    mf = 1.0 if cm == 0 else float(rm) / float(cm)
    if cf >= 1 or mf >= 1:
        return 0
    return int((1 - abs(cf - mf)) * 10)


def ref_le(l: float, r: float, diff: float) -> bool:            # resource_info.go:269-274
    return l < r or abs(l - r) < diff


def ref_less_equal(l, r) -> bool:                                # resource_info.go:268-302 on dense vectors
    if not ref_le(l[0], r[0], MIN_CPU) or not ref_le(l[1], r[1], MIN_MEM):
        return False
    for k in range(2, len(l)):
        if l[k] <= MIN_SCALAR:
            continue
        if not ref_le(l[k], r[k], MIN_SCALAR):
            return False
    return True


def ref_aff_score(count: int, mn: int, mx: int) -> int:         # interpod_affinity.go:222-228
    if mx - mn <= 0:
        return 0
    return int(10.0 * (float(count - mn) / float(mx - mn)))


def _with_hi(key: int, add: int) -> int:
    return (((key >> 32) + add) << 32 & MASK64) | (key & 0xFFFFFFFF)


def ref_add_pref_term(key: int, w: int, count: int, max_count: int) -> int:   # reduce.go:28-63 (NormalizeReduce(10, false)) * weight
    if key == 0 or max_count <= 0:
        return key
    return _with_hi(key, w * go_div(10 * count, max_count))


def ref_aff_add_score(key: int, w: int, score: int) -> int:
    return key if key == 0 else _with_hi(key, w * score)


# ---------------------------------------------------------------- cases
def capacities(rng, n_random=100_000):
    """1..16, an allocatable with system-reserved taken off, the float / int conversion edges, and log-uniform values up to 2^58
    with random low bits (most of them do not convert to float exactly)."""
    fixed = list(range(1, 17)) + [7910, 32879468 * 1024, 24 << 40]
    for p in (24, 31, 53):
        fixed += [(1 << p) - 1, 1 << p, (1 << p) + 1]
    fixed += [(1 << 58) - 1, 1 << 58]
    bits = rng.integers(1, 59, n_random)
    rand = rng.integers(np.int64(1) << (bits - 1), np.int64(1) << bits)
    return np.concatenate([np.array(fixed, dtype=np.int64), rand.astype(np.int64)])


def div_cases(seed=5, n_random=100_000):
    rng = np.random.default_rng(seed)
    b = capacities(rng, n_random)
    k = np.arange(11, dtype=np.int64)[None, :, None]
    d = np.arange(-2, 3, dtype=np.int64)[None, None, :]
    a = (k * b[:, None, None] + d).reshape(len(b), -1)
    bb = np.repeat(b, a.shape[1])
    a = a.reshape(-1)
    keep = (a >= 0) & (a <= 10 * bb)
    ra = rng.integers(0, 10 * b + 1)
    return np.concatenate([a[keep], ra]), np.concatenate([bb[keep], b])


def requested_cases(seed=6):
    rng = np.random.default_rng(seed)
    # above 2^58 the engine divides in int64 (up to 2^59: 10 * capacity still fits in int64, as in the reference)
    caps = np.concatenate([[0, (1 << 58) + 1, (1 << 59) + 12345], capacities(rng, 20_000)]).astype(np.int64)
    req, cap = [], []
    for c in caps.tolist():
        req += [0, max(c - 1, 0), c, c + 1, int(rng.integers(0, c + 1)), int(rng.integers(0, c + 1))]
        cap += [c] * 6
    return np.array(req, dtype=np.int64), np.array(cap, dtype=np.int64)


def balanced_cases(seed=7):
    rng = np.random.default_rng(seed)
    rows = []
    # every pair of fractions p/q with small denominators: many of them put (1 - |cf - mf|) * 10 within an ulp of an integer
    dens = [1, 2, 3, 4, 5, 7, 8, 10, 20, 100, 1000, 7910]
    for qc in dens:
        for qm in dens:
            for pc in range(0, qc + 1, max(1, qc // 20)):
                for pm in range(0, qm + 1, max(1, qm // 20)):
                    for sc, sm in ((1000, 1 << 30), (1, 1), (7, 32879468 * 1024)):
                        rows.append((pc * sc, qc * sc, pm * sm, qm * sm))
                        rows.append((pc * sc + 1, qc * sc, pm * sm, qm * sm))
                        rows.append((pc * sc, qc * sc, max(pm * sm - 1, 0), qm * sm))
    # capacity 0 on either axis, fractions >= 1, equal fractions
    for _ in range(20000):
        cc = int(rng.choice([0, 1, 7910, 32000, 1 << 40, int(rng.integers(1, 1 << 50))]))
        cm = int(rng.choice([0, 1, 32879468 * 1024, 24 << 40, int(rng.integers(1, 1 << 50))]))
        rc = int(rng.integers(0, int(cc * 1.3) + 2))
        rm = int(rng.integers(0, int(cm * 1.3) + 2))
        rows.append((rc, cc, rm, cm))
        if cc and cm:
            m = int(rng.integers(1, 1000))
            rows.append((rc, cc, rc * m, cc * m))                        # equal fractions
            rows.append((cc, cc, rm, cm))                                # cpu fraction exactly 1
    return np.array(rows, dtype=np.int64).T


def le_cases(seed=3):
    """The existing host test's vectors (the reference's LessEqual tests, every epsilon boundary, random values)."""
    eps = [10.0, 10.0 * 1024 * 1024]
    vals = [0.0, -0.0, 1.0, 4.0, 10.0, 2000.0, 4000.0, 8000.0, 1e9, 4e9, 10.0 * 1024 * 1024, 1e300, -1e300, 5e-324, -5e-324,
            9.999999999999998, 10.000000000000002]
    rng = np.random.default_rng(seed)
    cases = [(l, r, e) for l in vals for r in vals for e in eps]
    for e in eps:
        for base in (0.0, 1000.0, 3e9, 1e15, -9.0, -10.0 * 1024 * 1024 + 1):
            for d in (e, np.nextafter(e, 0), np.nextafter(e, 1e300), -e, -np.nextafter(e, 0), e / 2, 0.0, 1.0, -1.0):
                cases.append((base + d, base, e))
                cases.append((base, base + d, e))
    cases += [(float(a), float(b), float(e)) for a, b, e in zip(rng.integers(0, 1 << 40, 20000), rng.integers(0, 1 << 40, 20000),
                                                              rng.choice(eps, 20000))]
    cases += [(float(a), float(a + d), 10.0) for a, d in zip(rng.integers(-100000, 100000, 20000), rng.integers(-12, 13, 20000))]
    l, r, e = (np.array(x, dtype=np.float64) for x in zip(*cases))
    return l, r, e


def res_le_cases(R, seed=11, n=40000):
    rng = np.random.default_rng(seed + R)
    cpu = np.array([0.0, 1.0, 9.0, 10.0, 11.0, 1000.0, 7910.0])
    mem = np.array([0.0, 1.0, MIN_MEM - 1, MIN_MEM, MIN_MEM + 1, 1 << 30, 32879468.0 * 1024])
    sc = np.array([0.0, 1.0, 9.0, 10.0, 10.000000000000002, 11.0, 20.0, 1000.0])
    l = np.zeros((n, R))
    r = np.zeros((n, R))
    l[:, 0] = rng.choice(cpu, n)
    l[:, 1] = rng.choice(mem, n)
    l[:, 2:] = rng.choice(sc, (n, R - 2))
    # the right side: the left side plus a boundary offset, or an unrelated value
    off_c = rng.choice([0.0, -9.0, -10.0, -11.0, 1.0, -1000.0], n)
    off_m = rng.choice([0.0, -MIN_MEM + 1, -MIN_MEM, -MIN_MEM - 1, 1.0], n)
    off_s = rng.choice([0.0, -9.0, -10.0, -11.0, 1.0], (n, R - 2))
    r[:, 0] = np.where(rng.random(n) < 0.8, l[:, 0] + off_c, rng.choice(cpu, n))
    r[:, 1] = np.where(rng.random(n) < 0.8, l[:, 1] + off_m, rng.choice(mem, n))
    r[:, 2:] = np.where(rng.random((n, R - 2)) < 0.7, l[:, 2:] + off_s, rng.choice(sc, (n, R - 2)) * (rng.random((n, R - 2)) < 0.7))
    return l, r


def aff_cases(seed=13, n=60000):
    rng = np.random.default_rng(seed)
    mn = rng.choice([-(1 << 40), -1000, -7, 0, 3], n) + rng.integers(-5, 6, n)
    span = rng.choice([0, 0, 1, 3, 7, 10, 1000, 7910, (1 << 53) + 1, 1 << 58], n)
    mx = mn + span - (rng.random(n) < 0.05)               # max == min, and now and then max < min
    count = mn + (rng.random(n) * (span + 1)).astype(np.int64)
    count = np.where(rng.random(n) < 0.1, mx, count)
    count = np.where(rng.random(n) < 0.1, mn, count)
    return count.astype(np.int64), mn.astype(np.int64), mx.astype(np.int64)


def key_cases(seed=17, n=60000):
    rng = np.random.default_rng(seed)
    hi = rng.choice([0, 1, 5, 1 << 20, (1 << 31) - 1, 1 << 31, (1 << 32) - 2, (1 << 32) - 1], n) + rng.integers(-3, 4, n)
    hi = np.clip(hi, 0, (1 << 32) - 1).astype(np.uint64)
    lo = rng.choice([0, 1, 0xFFFFFFFF, 0xFFFFFFFE], n).astype(np.uint64)
    lo = np.where(rng.random(n) < 0.5, rng.integers(0, 1 << 32, n).astype(np.uint64), lo)
    key = (hi << np.uint64(32)) | lo
    key = np.where(rng.random(n) < 0.05, np.uint64(0), key)
    w = rng.choice([-100, -5, -1, 0, 1, 2, 5, 100, (1 << 31) - 1, -(1 << 31)], n).astype(np.int64)
    count = rng.integers(-300, 301, n)
    count = np.where(rng.random(n) < 0.2, rng.integers(-(1 << 40), 1 << 40, n), count).astype(np.int64)
    max_count = rng.choice([-1, 0, 1, 3, 7, 10, 300, 1 << 40], n).astype(np.int64)
    score = rng.integers(-20, 21, n).astype(np.int64)
    return key, w, count, max_count, score


# ---------------- eval_pair: packed node records (TileAcc layout) and a restatement of predicates.go + the three priorities
NODE_NOT_READY, NODE_NET_UNAVAILABLE, NODE_UNSCHEDULABLE = 1, 2, 4
NODE_MEM_PRESSURE, NODE_DISK_PRESSURE, NODE_PID_PRESSURE = 8, 16, 32
TASK_BEST_EFFORT = 1
TILE_NODES = 128


def random_pairs(seed, R, W, n):
    """n (conf-independent) pairs of (class, node): requests on the LessEqual boundaries of the node's Idle / Releasing, zero and
    irregular capacities, non-zero sums beyond allocatable, pod counts at the cap, sparse atom masks."""
    rng = np.random.default_rng(seed)
    nodes, classes = [], []
    for i in range(n):
        req = [float(rng.choice([0, 1, 10, 11, 100, 250, 1000, 1999, 7910]))]
        req.append(float(rng.choice([0, 1, 10 << 20, 200 << 20, 1 << 30, 3 << 30, 32879468 * 1024])))
        req += [float(rng.choice([0, 1, 10, 11, 1000, 2000])) for _ in range(R - 2)]
        def near(k):
            eps = MIN_MEM if k == 1 else 10.0
            choice = rng.integers(0, 6)
            if choice == 0:
                return req[k] + float(rng.choice([0.0, -eps + 1, -eps, -eps - 1, 1.0, -1.0]))
            if choice == 1:
                return float(rng.choice([-9.0, -1.0, 0.0])) if k != 1 else float(rng.choice([-MIN_MEM + 1, -1.0, 0.0]))
            return req[k] * float(rng.integers(0, 40)) + float(rng.integers(0, 3)) * (eps if k != 1 else 1.0)
        idle = [near(k) for k in range(R)]
        rel = [near(k) for k in range(R)]
        alloc_cpu = int(rng.choice([0, 1000, 7910, 32000, 96000, int(rng.integers(1, 1 << 20))]))
        alloc_mem = int(rng.choice([0, 32879468 * 1024, 128 << 30, 24 << 40, int(rng.integers(1, 1 << 45))]))
        nz_cpu = int(rng.choice([0, 100, alloc_cpu, alloc_cpu + 1, int(rng.integers(0, 2 * alloc_cpu + 2))]))
        nz_mem = int(rng.choice([0, 200 << 20, alloc_mem, alloc_mem + 1, int(rng.integers(0, 2 * alloc_mem + 2))]))
        max_pods = int(rng.choice([0, 1, 8, 110]))
        pods = max(0, max_pods - int(rng.choice([-1, 0, 1, 2, 50])))
        flags = 0
        for bit in (NODE_NOT_READY, NODE_NET_UNAVAILABLE, NODE_UNSCHEDULABLE, NODE_MEM_PRESSURE, NODE_DISK_PRESSURE, NODE_PID_PRESSURE):
            if rng.random() < 0.06:
                flags |= bit
        def mask(density):
            return [int(rng.integers(0, 1 << 63)) & int(rng.integers(0, 1 << 63)) if rng.random() < density else 0 for _ in range(W)]
        labels = [int(x) for x in rng.integers(0, 1 << 63, W)]
        taints = mask(0.15)
        ports = mask(0.2)
        nodes.append(dict(idle=idle, rel=rel, alloc_cpu=alloc_cpu, alloc_mem=alloc_mem, nz_cpu=nz_cpu, nz_mem=nz_mem, pods=pods,
                          max_pods=max_pods, flags=flags, labels=labels, taints=taints, ports=ports))
        def sub_of(words, p):      # a random subset of the node's labels, or (now and then) a bit it lacks
            out = []
            for x in words:
                m = x & int(rng.integers(0, 1 << 63)) & int(rng.integers(0, 1 << 63)) & int(rng.integers(0, 1 << 63))
                if rng.random() < p:
                    m |= 1 << int(rng.integers(0, 64))
                out.append(m)
            return out
        n_aff = int(rng.choice([0, 0, 1, 2, 4]))
        aff = [sub_of(labels, 0.3) if t < n_aff else [0] * W for t in range(KB_MAX_AFF_TERMS)]
        tol = [x | (int(rng.integers(0, 1 << 63)) if rng.random() < 0.3 else 0) for x in (taints if rng.random() < 0.8 else [0] * W)]
        classes.append(dict(initreq=req, nz_cpu=int(rng.choice([100, int(req[0]), 0])), nz_mem=int(rng.choice([200 << 20, int(req[1]), 0])),
                            sel_req=sub_of(labels, 0.1) if rng.random() < 0.5 else [0] * W, aff=aff, n_aff=n_aff, tol=tol,
                            port_conflict=mask(0.2), flags=TASK_BEST_EFFORT if rng.random() < 0.3 else 0))
    return nodes, classes


def pack_tiles(nodes, R, W):
    ncols = 2 * R + 6 + 3 * W
    nt = (len(nodes) + TILE_NODES - 1) // TILE_NODES
    t = np.zeros((max(nt, 1), ncols, TILE_NODES), dtype=np.uint64)
    f64 = lambda x: np.array([x], dtype=np.float64).view(np.uint64)[0]
    u64 = lambda x: np.uint64(x & MASK64)
    for i, n in enumerate(nodes):
        tile, j = divmod(i, TILE_NODES)
        col = t[tile]
        for k in range(R):
            col[k, j] = f64(n["idle"][k])
            col[R + k, j] = f64(n["rel"][k])
        col[2 * R, j] = u64(n["alloc_cpu"])
        col[2 * R + 1, j] = u64(n["alloc_mem"])
        col[2 * R + 2, j] = u64(n["nz_cpu"])
        col[2 * R + 3, j] = u64(n["nz_mem"])
        col[2 * R + 4, j] = u64(n["pods"] | (n["max_pods"] << 32))
        col[2 * R + 5, j] = u64(n["flags"])
        for w in range(W):
            col[2 * R + 6 + w, j] = u64(n["labels"][w])
            col[2 * R + 6 + W + w, j] = u64(n["taints"][w])
            col[2 * R + 6 + 2 * W + w, j] = u64(n["ports"][w])
    return np.ascontiguousarray(t.reshape(-1))


def class_rec(c, R, W):
    rec = ClassRec()
    for k in range(R):
        rec.initreq[k] = c["initreq"][k]
        rec.resreq[k] = c["initreq"][k]
    rec.nz_cpu, rec.nz_mem = c["nz_cpu"], c["nz_mem"]
    for w in range(W):
        rec.sel_req[w] = c["sel_req"][w]
        rec.tol[w] = c["tol"][w]
        rec.port_conflict[w] = c["port_conflict"][w]
        for t in range(KB_MAX_AFF_TERMS):
            rec.aff[t][w] = c["aff"][t][w]
    rec.n_aff = c["n_aff"]
    rec.flags = c["flags"]
    return rec


def ref_eval_pair(cf: EvalConf, c, n, idx):
    """(key, fits_idle, pred_ok) of one pair, from the reference: allocate.go:73-87 (+ backfill.go:50-65 / node_info.go:161-167),
    predicates.go:122-265 and the vendored predicates, the least / most requested and balanced priorities, scheduler_helper.go:162-168."""
    R, W = cf.R, cf.W
    fi = ref_less_equal(c["initreq"][:R], n["idle"][:R])
    fr = ref_less_equal(c["initreq"][:R], n["rel"][:R])
    ok = {0: fi or fr, 1: fi, 2: True}[cf.fit_mode]
    pok = True
    if cf.predicates:
        if n["max_pods"] <= n["pods"]:
            pok = False
        if n["flags"] & (NODE_NOT_READY | NODE_NET_UNAVAILABLE | NODE_UNSCHEDULABLE):
            pok = False
        for w in range(W):
            if n["labels"][w] & c["sel_req"][w] != c["sel_req"][w]:
                pok = False                     # PodMatchNodeSelector: a nodeSelector entry the node lacks
            if n["ports"][w] & c["port_conflict"][w]:
                pok = False                     # PodFitsHostPorts
            if n["taints"][w] & ~c["tol"][w]:
                pok = False                     # PodToleratesNodeTaints
        if c["n_aff"]:                          # required node affinity: OR over the terms, each an AND of requirements
            if not any(all(n["labels"][w] & c["aff"][t][w] == c["aff"][t][w] for w in range(W)) for t in range(c["n_aff"])):
                pok = False
        if cf.mem_pressure and (c["flags"] & TASK_BEST_EFFORT) and (n["flags"] & NODE_MEM_PRESSURE):
            pok = False
        if cf.disk_pressure and (n["flags"] & NODE_DISK_PRESSURE):
            pok = False
        if cf.pid_pressure and (n["flags"] & NODE_PID_PRESSURE):
            pok = False
    if not (ok and pok):
        return 0, fi, pok
    score = cf.score_bias
    if cf.nodeorder:
        rc, rm = n["nz_cpu"] + c["nz_cpu"], n["nz_mem"] + c["nz_mem"]
        ac, am = n["alloc_cpu"], n["alloc_mem"]
        score += go_div(ref_least(rc, ac) + ref_least(rm, am), 2) * cf.w_least
        score += go_div(ref_most(rc, ac) + ref_most(rm, am), 2) * cf.w_most
        score += ref_balanced(rc, ac, rm, am) * cf.w_balanced
    return ((score << 32) & MASK64) | (0xFFFFFFFF - idx), fi, pok


def eval_confs(R, W):
    out = []
    for predicates, nodeorder, (wl, wm, wb), fit_mode, press in [
            (1, 1, (1, 0, 1), 0, (0, 0, 0)), (1, 1, (0, 3, 2), 0, (1, 1, 1)), (1, 1, (-2, 0, 1), 1, (1, 0, 1)),
            (0, 1, (1, 1, 1), 0, (0, 0, 0)), (1, 0, (1, 0, 1), 2, (0, 1, 0)), (0, 0, (0, 0, 0), 1, (0, 0, 0))]:
        cf = EvalConf(R=R, W=W, predicates=predicates, mem_pressure=press[0], disk_pressure=press[1], pid_pressure=press[2],
                      nodeorder=nodeorder, w_least=wl, w_most=wm, w_balanced=wb, score_bias=40, fit_mode=fit_mode)
        out.append(cf)
    return out


EVAL_GEOMETRIES = [(1, 3, 2), (0, 3, 2), (0, 2, 1), (0, 5, 3)]     # (1 = eval_pair<3,2> / 0 = eval_pair<0,0>, R, W)


# ---------------------------------------------------------------- the checks, shared with the GPU file (device = 1)
def _first_bad(got, exp, *inputs):
    bad = np.nonzero(np.asarray(got) != np.asarray(exp))[0]
    if len(bad):
        i = int(bad[0])
        raise AssertionError(f"{len(bad)} case(s) differ; first: inputs {[x[i] for x in inputs]} got {got[i]} expected {exp[i]}")


def check_div(device):
    a, b = div_cases()
    got = run_div(device, a, b)
    _first_bad(got, a // b, a, b)                        # non-negative: numpy's floor division is Go's truncation


def check_requested(device):
    req, cap = requested_cases()
    for which, ref in (("least", ref_least), ("most", ref_most)):
        got = run_requested(device, which, req, cap)
        exp = np.array([ref(int(r), int(c)) for r, c in zip(req, cap)], dtype=np.int64)
        _first_bad(got, exp, req, cap)


def check_balanced(device):
    rc, cc, rm, cm = balanced_cases()
    got = run_balanced(device, rc, cc, rm, cm)
    exp = np.array([ref_balanced(*map(int, x)) for x in zip(rc, cc, rm, cm)], dtype=np.int64)
    _first_bad(got, exp, rc, cc, rm, cm)
    # the fixture does reach the integer boundary from below (and the rounding then decides)
    v = [(1 - abs((float(a) / float(b) if b else 1.0) - (float(c) / float(d) if d else 1.0))) * 10 for a, b, c, d in zip(rc, cc, rm, cm)]
    assert sum(1 for x in v if 0 < x < 10 and x != math.floor(x) and math.ceil(x) - x < 1e-14) > 50


def check_le(device):
    l, r, e = le_cases()
    got = run_le(device, l, r, e)
    exp = np.array([ref_le(a, b, d) for a, b, d in zip(l.tolist(), r.tolist(), e.tolist())])
    _first_bad(got, exp, l, r, e)
    for R in (3, 5):
        L, Rr = res_le_cases(R)
        got = run_res_le(device, L, Rr)
        exp = np.array([ref_less_equal(x.tolist(), y.tolist()) for x, y in zip(L, Rr)])
        _first_bad(got, exp, L, Rr)
        assert 0.05 < exp.mean() < 0.9


def check_aff(device):
    count, mn, mx = aff_cases()
    got = run_aff_score(device, count, mn, mx)
    exp = np.array([ref_aff_score(int(c), int(a), int(b)) for c, a, b in zip(count, mn, mx)], dtype=np.int64)
    _first_bad(got, exp, count, mn, mx)
    key, w, cnt, maxc, score = key_cases()
    got = run_add_pref_term(device, key, w, cnt, maxc)
    exp = np.array([ref_add_pref_term(int(k), int(a), int(b), int(c)) for k, a, b, c in zip(key, w, cnt, maxc)], dtype=np.uint64)
    _first_bad(got, exp, key, w, cnt, maxc)
    w32 = np.clip(w, -(1 << 31), (1 << 31) - 1)
    got = run_aff_add_score(device, key, w32, score)
    exp = np.array([ref_aff_add_score(int(k), int(a), int(s)) for k, a, s in zip(key, w32, score)], dtype=np.uint64)
    _first_bad(got, exp, key, w32, score)


def check_eval_pair(device, geometry, R, W, seed=23, n=3000):
    nodes, classes = random_pairs(seed + 100 * R + W, R, W, n)
    tiles = pack_tiles(nodes, R, W)
    recs = [class_rec(c, R, W) for c in classes]
    seen_fi = seen_key = seen_pok = 0
    for cf in eval_confs(R, W):
        key, fi, pok = run_eval_pair(device, geometry, cf, recs, tiles)
        for i in range(n):
            ek, efi, epok = ref_eval_pair(cf, classes[i], nodes[i], i)
            assert (int(key[i]), bool(fi[i]), bool(pok[i])) == (ek, efi, epok), \
                (f"eval_pair geometry {geometry} R{R} W{W} conf {[getattr(cf, f) for f, _ in cf._fields_]} pair {i}: "
                 f"got {(hex(int(key[i])), bool(fi[i]), bool(pok[i]))} expected {(hex(ek), efi, epok)}\nnode {nodes[i]}\nclass {classes[i]}")
        seen_fi += int(fi.sum())
        seen_key += int((key != 0).sum())
        seen_pok += int(pok.sum())
    total = n * len(eval_confs(R, W))
    assert 0.1 * total < seen_fi < 0.9 * total and 0.1 * total < seen_key < 0.9 * total and 0.1 * total < seen_pok < 0.95 * total


# ---------------------------------------------------------------- host build
def test_probe_mirrors_the_engine_structs():
    L = probe()
    assert L.kbp_sizeof_class_rec() == C.sizeof(ClassRec)
    assert L.kbp_sizeof_eval_conf() == C.sizeof(EvalConf)
    assert L.kbp_tile_nodes() == TILE_NODES


def test_div_0_to_10_host_build_is_exact():
    check_div(0)


def test_least_and_most_requested_host_build():
    check_requested(0)


def test_balanced_score_host_build():
    check_balanced(0)


def test_le_func_and_res_less_equal_host_build():
    check_le(0)


def test_affinity_scores_host_build():
    check_aff(0)


@pytest.mark.parametrize("geometry,R,W", EVAL_GEOMETRIES)
def test_eval_pair_host_build(geometry, R, W):
    check_eval_pair(0, geometry, R, W)
