"""NestedQuery in the references (tests/nested_reference.py), on the CPU: the object-level reference pinned to the hit sets of
the reference project's ObjectFieldDefTest (its initIndex, registerFieldsObject.json: pickup_partners is the one nested
field, so every document is a block of its pickup_partners children and the parent), then to hand-computed floats of
every score mode, and the array-level reference over compile_tree held to the same answers."""
import numpy as np
import pytest

import nested_reference as nr
import phrase_reference as pr
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, NestedQuery, Occur, RangeQuery, TermQuery)

S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
F32 = np.float32

# ---------------------------------------------------------------- ObjectFieldDefTest's index
# fields: 0 pickup_partners.name, 1 delivery_areas.partner.partner_name (flattened object), 2 _nested_path
NAMES = ["AAA", "BBB", "CCC", "EEE", "FFF", "GGG"]
PARTNERS = ["efg", "567"]
T = {("name", n): i for i, n in enumerate(NAMES)}
T.update({("partner", p): len(NAMES) + i for i, p in enumerate(PARTNERS)})
ROOT, PICKUP = len(T), len(T) + 1
TERM_FIELD = [0] * len(NAMES) + [1] * len(PARTNERS) + [2, 2]


def object_index(update=False, delete=False):
    """initIndex's documents as blocks (children first); update: doc_id 5 (real_id 3) re-added with child FFF, which deletes
    the parent of real_id 3 (its child stays: the update deletes by the id term, which only the parent holds); delete:
    the parent of doc_id 4 deleted. Returns (shard, {parent doc: doc_id})."""
    blocks = [(1, ["AAA", "BBB"], "efg"), (2, ["AAA", "CCC"], "567"), (3, ["EEE"], None), (4, ["GGG"], None)]
    if update:
        blocks.append((5, ["FFF"], None))
    docs, ids = [], {}
    for doc_id, kids, partner in blocks:
        for k in kids:
            docs.append([[[T["name", k]]], [], [[PICKUP]]])
        ids[len(docs)] = doc_id
        docs.append([[], [[T["partner", partner]]] if partner else [], [[ROOT]]])
    sh = pr.shard_from_tokens(docs, TERM_FIELD, 3)
    sh.parent_term = ROOT
    live = np.ones(sh.n_docs, np.uint8)
    for p, doc_id in ids.items():
        if (update and doc_id == 3) or (delete and doc_id == 4):
            live[p] = 0
    sh.live_docs = live
    return sh, ids


def root_filtered(q):
    """the filter the reference puts on every top-level query of an index with nested fields"""
    return BooleanQuery().add(TermQuery(ROOT), F).add(q, M)


def nested(name, mode="none"):
    return NestedQuery(TermQuery(T["name", name]), PICKUP, mode)


def hits(sh, ids, q):
    d, s, c, t = nr.NestedReference(sh).search([root_filtered(q)], 10)
    d2, s2, c2, t2, _ = nr.search(sh, [root_filtered(q)], 10)
    assert np.array_equal(d, d2) and np.array_equal(s.view(np.uint32), s2.view(np.uint32)) and np.array_equal(c, c2[:1])
    return sorted(ids[int(x)] for x in d[0, :c[0]])


def test_simple_nested_docs():
    sh, ids = object_index()
    assert hits(sh, ids, nested("BBB")) == [1]


def test_combined_nested_query():
    sh, ids = object_index()
    q = BooleanQuery().add(nested("AAA"), M).add(TermQuery(T["partner", "567"]), M)
    assert hits(sh, ids, q) == [2]
    assert hits(sh, ids, nested("AAA")) == [1, 2]


def test_update_nested_object():
    sh, ids = object_index()
    assert hits(sh, ids, nested("EEE")) == [3]
    sh, ids = object_index(update=True)
    assert hits(sh, ids, nested("EEE")) == []
    assert hits(sh, ids, nested("FFF")) == [5]


def test_delete_nested_object():
    sh, ids = object_index()
    assert hits(sh, ids, nested("GGG")) == [4]
    sh, ids = object_index(delete=True)
    assert hits(sh, ids, nested("GGG")) == []


# ---------------------------------------------------------------- hand-computed floats
# One text field and the path field; doc values column 0 numbers the docs, so a child query of SHOULD ranges, one per
# child and each of one doc, scores every child exactly its range's boost.
LEAF, ROOT2, PATH = 0, 1, 2


def block_shard(blocks, trailing=0, parent_on_path=()):
    """blocks: the child count of each block; trailing: children after the last parent; parent_on_path: parents (block
    indexes) that also hold the path term"""
    docs, parents = [], []
    for b, n in enumerate(blocks):
        docs += [[[[LEAF]], [[PATH]]] for _ in range(n)]
        parents.append(len(docs))
        docs.append([[[LEAF]], [[ROOT2, PATH]] if b in parent_on_path else [[ROOT2]]])
    docs += [[[[LEAF]], [[PATH]]] for _ in range(trailing)]
    sh = pr.shard_from_tokens(docs, [0, 1, 1], 2)
    sh.columns = [np.arange(sh.n_docs, dtype=np.int64)]
    sh.column_has = [None]
    sh.parent_term = ROOT2
    return sh, parents


def scored_children(scores):
    """a child query that scores doc d exactly scores[d] (float32), docs without a score not matching"""
    q = BooleanQuery()
    for d, s in scores.items():
        q.add(BoostQuery(RangeQuery(0, d, d), float(s)), S)
    return q


def page(sh, q):
    d, s, c, t = nr.NestedReference(sh).search([q], 20)
    d2, s2, c2, t2, _ = nr.search(sh, [q], 20)
    assert np.array_equal(d, d2) and np.array_equal(s.view(np.uint32), s2.view(np.uint32)) and np.array_equal(t, t2)
    return dict(zip(d[0, :c[0]].tolist(), s[0, :c[0]].tolist())), int(t[0])


@pytest.mark.parametrize("mode", ["none", "sum", "avg", "max", "min"])
def test_modes(mode):
    sh, (p0, p1) = block_shard([3, 2])
    sc = {0: F32(1.0), 1: F32(2.0 ** -24), 2: F32(2.0 ** -24), 4: F32(0.25), 5: F32(3.5)}   # (doc 3 is the first parent)
    got, total = page(sh, NestedQuery(scored_children(sc), PATH, mode))
    want = {"none": (F32(0), F32(0)),
            # double sum in child order: 1 + 2^-23 (a float sum would stay at 1.0)
            "sum": (F32(1.0 + 2.0 ** -23), F32(3.75)),
            "avg": (F32((1.0 + 2.0 ** -23) / 3), F32(3.75 / 2)),
            "max": (F32(1.0), F32(3.5)),
            "min": (F32(2.0 ** -24), F32(0.25))}[mode]
    assert total == 2 and got == {p0: want[0], p1: want[1]}
    if mode == "sum":
        f = F32(0)
        for d in (0, 1, 2):
            f = F32(f + sc[d])
        assert f == F32(1.0) != want[0]


def test_avg_divides_in_double():
    sh, (p0,) = block_shard([3])
    got, _ = page(sh, NestedQuery(scored_children({0: 1.0, 1: 1.0, 2: 0.7}), PATH, "avg"))
    f = F32(F32(F32(1.0) + F32(1.0)) + F32(0.7))
    assert got == {p0: F32(0.9)} and F32(f / F32(3)) != F32(0.9)   # (float)(2.7f as double / 3), not a float division


def test_boosts_fold_through_the_join():
    sh, (p0,) = block_shard([2])
    q = BoostQuery(NestedQuery(BoostQuery(scored_children({0: 1.5, 1: 0.5}), 2.0), PATH, "sum"), 3.0)
    got, _ = page(sh, q)
    assert got == {p0: F32(F32(3.0) * F32(2.0) * F32(1.5)) + F32(F32(3.0) * F32(2.0) * F32(0.5))}


def test_deleted_child_of_live_parent_joins():
    sh, (p0, p1) = block_shard([2, 1])
    live = np.ones(sh.n_docs, np.uint8)
    live[0] = 0          # a deleted child: still joins
    live[p1] = 0         # a deleted parent: no hit
    sh.live_docs = live
    got, total = page(sh, NestedQuery(scored_children({0: 1.0, 1: 2.0, 3: 4.0}), PATH, "sum"))
    assert got == {p0: F32(3.0)} and total == 1


def test_child_that_is_a_parent_and_trailing_children():
    sh, (p0, p1) = block_shard([1, 1], trailing=2, parent_on_path=(0,))
    n = sh.n_docs
    # p0 holds the path term and matches the child query: it joins nothing (and its child still joins p0)
    got, total = page(sh, NestedQuery(scored_children({0: 1.0, p0: 8.0, n - 1: 16.0, n - 2: 32.0}), PATH, "sum"))
    assert got == {p0: F32(1.0)} and total == 1
    # only the parent and the trailing children match: nothing joins
    got, total = page(sh, NestedQuery(scored_children({p0: 8.0, n - 1: 16.0}), PATH, "max"))
    assert got == {} and total == 0


def test_join_under_every_occur():
    sh, (p0, p1) = block_shard([1, 1])
    j = NestedQuery(scored_children({0: 2.0}), PATH, "max")
    other = TermQuery(LEAF)
    ref = nr.NestedReference(sh)
    _, leaf_s = ref.eval(other)
    got, _ = page(sh, BooleanQuery().add(j, M).add(other, S))
    assert got == {p0: F32(2.0) + leaf_s[p0]}
    got, _ = page(sh, BooleanQuery().add(j, F).add(other, S))
    assert got == {p0: leaf_s[p0]}
    got, _ = page(sh, BooleanQuery().add(j, N).add(TermQuery(ROOT2), S))
    assert list(got) == [p1]
