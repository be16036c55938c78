"""CPU check of GLCM phase A's MCC classification (glcm_fast_angle, compiled for the host from the device header by
tests/host_emul/glcm_full_emul.cpp) against the numpy restatement in tests/mcc_class.py, and of that restatement against
the window oracle (helpers.mcc_angle).

A level graph on nlev nodes with at most nlev - 1 distinct edges (self-loops included) is disconnected or a tree; phase A
settles such graphs by counting (MCC 1), and the rest by its connectivity sweep and 2-colouring.  Every route is
exercised here."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import adversarial_windows, corpus_window, mcc_angle
from mcc_class import BIPARTITE, EMPTY, ONE, SPLIT, TASK, classify
from pyradiomics_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
G_MCC = 19                       # MCC in the library's GLCM feature order


@pytest.fixture(scope="module")
def emul():
    so = os.path.join(HERE, "host_emul", "libglcm_full_emul.so")
    src = os.path.join(HERE, "host_emul", "glcm_full_emul.cpp")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so + ".%d" % os.getpid(), src])
    os.replace(so + ".%d" % os.getpid(), so)
    lib = C.CDLL(so)
    lib.emul_glcm_angle.restype = C.c_longlong
    return lib


def _windows(rng, count):
    """i.i.d. windows over 2 to 32 levels, a fifth of them with holes, plus the helpers' structured corpus"""
    ng = rng.integers(2, 33, (count, 1))
    w = rng.integers(1, 33, (count, 27)) % ng + 1
    holed = rng.random(count) < 0.2
    w[holed] *= rng.random((int(holed.sum()), 27)) > 0.3
    corpus = [corpus_window(rng, it) for it in range(count)] + adversarial_windows()
    return np.concatenate([w, np.array(corpus, np.int64)]).astype(np.uint8)


def test_restatement_matches_window_oracle():
    rng = np.random.default_rng(7)
    W = _windows(rng, 1500)
    for slot in range(13):
        cls, nlev, _, _ = classify(W, slot)
        for k, w in enumerate(W):
            r = mcc_angle(w, slot)
            if r is None:
                assert cls[k] == EMPTY
                continue
            want = ONE if r[1] == 1 else SPLIT if not r[2] else BIPARTITE if r[3] else TASK
            assert (cls[k], nlev[k]) == (want, r[1]), (w, slot)


def test_phase_a_classification_equals_restatement(emul):
    rng = np.random.default_rng(8)
    W = _windows(rng, 4000)
    s = _lib.make_settings(32, 32)
    # graphs settled by the edge count (disconnected / trees), and those left to the sweep (disconnected / bipartite
    # with a cycle / eigen-tasks)
    seen = dict.fromkeys(("split counted", "tree counted", "split swept", "bipartite swept", "task"), 0)
    for slot in range(13):
        cls, nlev, _, edges = classify(W, slot)
        counted = (nlev >= 2) & (edges < nlev)
        assert ((cls[counted] == SPLIT) | (cls[counted] == BIPARTITE)).all()
        seen["split counted"] += int((counted & (cls == SPLIT)).sum())
        seen["tree counted"] += int((counted & (cls == BIPARTITE)).sum())
        seen["split swept"] += int((~counted & (cls == SPLIT)).sum())
        seen["bipartite swept"] += int((~counted & (cls == BIPARTITE)).sum())
        seen["task"] += int((cls == TASK).sum())
        for k, w in enumerate(W):
            wp = np.ascontiguousarray(w).ctypes.data_as(C.c_void_p)
            for full in ((0, 1) if w.all() else (0,)):
                sums = np.zeros(24)
                tcls = C.c_ulonglong(0)
                tasks = emul.emul_glcm_angle(wp, slot, full, C.byref(s), sums.ctypes.data_as(C.c_void_p), C.byref(tcls))
                assert tasks >= 0
                want_task = cls[k] == TASK
                assert bool(tasks >> slot & 1) == want_task, (w, slot, cls[k])
                mcc = {EMPTY: 0.0, ONE: 0.0, SPLIT: 1.0, BIPARTITE: 1.0, TASK: 0.0}[int(cls[k])]
                assert sums[G_MCC] == mcc, (w, slot, cls[k])
                if want_task:
                    n = int(nlev[k])
                    assert tcls.value >> (4 * slot) & 15 == (0 if n <= 2 else 15 if n >= 17 else n - 2)
    assert min(seen.values()) > 500, seen


def test_edge_count_cases(emul):
    """hand-made body-diagonal graphs (slot 9, angle (1, 1, 1): pairs (p, p + 13) for p in {0, 1, 3, 4, 9, 10, 12, 13}):
    eight pairs of distinct levels (15 levels, 8 edges: counted); a triangle beside an edge with a self-loop (5 levels,
    5 distinct edges: the sweep finds two components); a triangle with a pendant level (4 levels, 4 edges, connected and
    not bipartite: an eigen-task, which one more counted edge would have hidden)"""
    s = _lib.make_settings(32, 32)
    pa = [0, 1, 3, 4, 9, 10, 12, 13]
    cases = []
    w = np.full(27, 30, np.uint8)                    # unpaired positions: a level no pair sees
    for k, p in enumerate(pa):
        w[p], w[p + 13] = 1 + 2 * k, 2 + 2 * k
    w[13] = 2                                        # p = 13 is the upper end of p = 0 and the lower end of 13 -> 26
    cases.append((w, True))
    w = np.full(27, 30, np.uint8)
    edges = [(1, 2), (2, 3), (3, 1), (4, 5)]
    for k, p in enumerate(pa):
        if p == 13:
            continue
        a, b = edges[k % 4]
        w[p], w[p + 13] = a, b
    w[26] = w[13]                                    # 13 -> 26 is (2, 2): a self-loop
    cases.append((w, False))
    w = np.full(27, 30, np.uint8)
    edges = [(1, 2), (2, 3), (3, 1), (3, 4)]
    for k, p in enumerate(pa):
        if p == 13:
            continue
        a, b = edges[k % 4]
        w[p], w[p + 13] = a, b
    w[26] = 1                                        # 13 -> 26 is (2, 1): no new level pair
    cases.append((w, False))
    for k, (w, counted) in enumerate(cases):
        cls, nlev, n, e = classify(w[None], 9)
        assert cls[0] == (TASK if k == 2 else SPLIT) and bool(e[0] < nlev[0]) == counted, (w, cls, nlev, n, e)
        for full in (0, 1):
            sums = np.zeros(24)
            tcls = C.c_ulonglong(0)
            tasks = emul.emul_glcm_angle(np.ascontiguousarray(w).ctypes.data_as(C.c_void_p), 9, full, C.byref(s),
                                         sums.ctypes.data_as(C.c_void_p), C.byref(tcls))
            assert (tasks, sums[G_MCC]) == ((1 << 9, 0.0) if k == 2 else (0, 1.0)), k
