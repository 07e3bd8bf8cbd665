"""Which sweep warm-ups the planner marks exact (WorkPlan::warm_exact, read back through the g++ planner harness
tests/csrc/warm_plan_harness.cpp, the batch planner harness with one more export): in
TOP_SCORES, a pure disjunction of two or more lists with a sweep warm-up whose term slots other than the warm-up's all
have a tf plane. The
marked slot is the sweep item's slot; the work list is the one an unmarked plan would have."""
import contextlib
import ctypes as C
import os

import numpy as np

import plan_harness as ph
from nrtsearch_b200.search import BooleanQuery, Occur, ScoreDoc, TermQuery

_WARM_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libwarm_plan_harness.so")


@contextlib.contextmanager
def warm_plan(d, qs, top_k, threshold, **kw):
    """ph.plan through libwarm_plan_harness.so; yields (plan, warm_exact per query). The plan is freed on exit, by the
    library that made it."""
    saved = ph._lib, ph._PATH
    ph._lib, ph._PATH = None, _WARM_PATH
    try:
        h = ph.lib()
        h.ph_warm_exact.argtypes = [C.c_void_p, C.c_void_p]
        p = ph.plan(d, qs, top_k, threshold, **kw)
        try:
            out = np.full(len(qs), -1, np.int32)
            if p.n_slices:
                h.ph_warm_exact(p._h, out.ctypes.data)
            yield p, out
        finally:
            p.close()
    finally:
        ph._lib, ph._PATH = saved

INT_MAX = ph.INT_MAX
N_DOCS = 1_000_000   # above the warm-up minimum; lists of >= N_DOCS / 64 = 15,625 postings get tf planes
# term: postings (the rarest list has the highest bound: term_max_x is 1.0 everywhere)
LENS = {"RARE": 5_000, "RARE2": 3_000, "P1": 100_000, "P2": 200_000, "NOPLANE": 10_000, "TINY": 15}


def _dict():
    names = list(LENS)
    off = np.zeros(len(names) + 1, np.int64)
    np.cumsum([LENS[n] for n in names], out=off[1:])
    return ph.Dictionary(N_DOCS, off), {n: i for i, n in enumerate(names)}


def _disj(*terms):
    q = BooleanQuery()
    for t in terms:
        q.add(TermQuery(int(t)), Occur.SHOULD)
    return q


def test_exact_warm_ups_are_marked_by_the_planes_of_the_other_slots():
    d, t = _dict()
    tp, _ = ph.index_rules(N_DOCS, d.term_off)
    assert [n for n in LENS if tp[t[n]] >= 0] == ["P1", "P2"]
    qs = [_disj(t["RARE"], t["P1"], t["P2"]),        # every other slot has a plane: exact, slot 0
          _disj(t["P1"], t["RARE2"]),                 # exact, slot 1
          _disj(t["RARE2"], t["NOPLANE"], t["P1"]),   # NOPLANE is not the warm-up's list and has no plane
          _disj(t["RARE"]),                           # one list: a lower-bound warm-up
          _disj(t["TINY"], t["P1"]),                  # 15 postings < 2 * top_k: no sweep warm-up
          _disj(t["P2"], t["RARE"])]                  # exact, slot 1
    want = [0, 1, -1, -1, -1, 1]
    with warm_plan(d, qs, 10, 1000) as (p, exact):
        assert exact.tolist() == want
        sweep = {int(q): ph.decode(w)[4] for q, w in zip(p.work_query, p.work_item) if ph.decode(w)[3] & ph.ITEM_SWEEP}
        items = p.work_query.tolist(), p.work_item.tolist()
    assert sorted(sweep) == [0, 1, 2, 3, 5]
    assert all(sweep[q] == s for q, s in enumerate(want) if s >= 0)
    # ScoreMode.COMPLETE: no exact warm-ups, the same work list
    with warm_plan(d, qs, 10, INT_MAX) as (c, exact):
        assert (exact == -1).all()
        assert (c.work_query.tolist(), c.work_item.tolist()) == items
    # searchAfter: no sweep warm-up at all
    with warm_plan(d, qs, 10, 1000, search_after=[ScoreDoc(0, 1.0)] * len(qs)) as (_, exact):
        assert (exact == -1).all()
