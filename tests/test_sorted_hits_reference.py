"""tests/sorted_hits_reference.py pinned to TopHitsCollectorManagerTest's known answers (testTopHitsRelevance,
testTopHitsStartHit, testTopHitsSort) and to hand-computed orders: ties by global doc, missing values, MIN / MAX selectors,
DOCID, a leading score with and without reverse, and 8 fields. CPU only."""
from types import SimpleNamespace

import numpy as np

import sorted_hits_reference as ref

COLUMN, DOCID, SCORE = 1, 2, 3


def known_answer_index():
    """TopHitsCollectorManagerTest's 100 docs (doc_id = id, int_field = 100 - id, int_field_2 = id, value = id + 2), added
    in shuffled order in segments of 10; the query scores int_field_2 * 3 (a FunctionScoreQuery script)"""
    ids = np.random.default_rng(7).permutation(100)
    sh = SimpleNamespace(doc_base=0, columns=[100 - ids, ids.copy(), ids + 2], column_has=[None, None, None], column_offsets=[])
    return sh, ids, (3 * ids).astype(np.float32)


def test_top_hits_relevance():
    sh, ids, scores = known_answer_index()
    docs, vals = ref.top_hits(sh, np.arange(100), scores, None, 5, 0)
    assert vals is None
    assert ids[docs].tolist() == [99, 98, 97, 96, 95]
    assert scores[docs].tolist() == [297, 294, 291, 288, 285]


def test_top_hits_start_hit():
    sh, ids, scores = known_answer_index()
    docs, _ = ref.top_hits(sh, np.arange(100), scores, None, 10, 5)
    assert ids[docs].tolist() == [94, 93, 92, 91, 90]
    assert scores[docs].tolist() == [282, 279, 276, 273, 270]


def test_top_hits_sort():
    sh, ids, scores = known_answer_index()
    docs, vals = ref.top_hits(sh, np.arange(100), scores, [(COLUMN, 0, 0, 0, 0)], 5, 0)
    assert ids[docs].tolist() == [99, 98, 97, 96, 95]
    assert vals[:, 0].tolist() == [1, 2, 3, 4, 5]


def small():
    """8 docs at doc_base 100: c0 with ties and missing docs, c1 multi-valued (offsets), c2 all equal"""
    c0 = np.array([5, 3, 5, -1, 3, 9, 5, 0], np.int64)
    has0 = np.array([1, 1, 1, 1, 1, 0, 1, 0], np.uint8)
    c1 = np.array([4, 8, 1, 7, 2, 6, 9], np.int64)            # doc 0: 4 8 | 1: 1 7 | 2: - | 3: 2 | 4: 6 9 | 5..7: -
    off1 = np.array([0, 2, 4, 4, 5, 7, 7, 7, 7], np.int64)
    return SimpleNamespace(doc_base=100, columns=[c0, c1, np.zeros(8, np.int64)], column_has=[has0, None, None],
                           column_offsets=[None, off1, None])


ALL = np.arange(8)
SC = np.array([2.0, 1.0, 2.0, 3.0, 1.0, 2.0, 0.5, 3.0], np.float32)


def test_ties_go_to_the_smaller_global_doc():
    sh = small()
    docs, vals = ref.top_hits(sh, ALL, SC, [(COLUMN, 2, 0, 0, 0)], 8, 0)
    assert docs.tolist() == list(range(100, 108)) and not vals.any()
    docs, _ = ref.top_hits(sh, ALL, SC, [(COLUMN, 2, 1, 0, 0)], 8, 0)   # reverse does not reverse the doc tie-break
    assert docs.tolist() == list(range(100, 108))
    docs, _ = ref.top_hits(sh, ALL, SC, None, 8, 0)                     # by score: equal scores by doc
    assert docs.tolist() == [103, 107, 100, 102, 105, 101, 104, 106]


def test_missing_values():
    sh = small()
    docs, vals = ref.top_hits(sh, ALL, SC, [(COLUMN, 0, 0, 0, 4)], 8, 0)   # docs 5 and 7 sort as 4
    assert docs.tolist() == [103, 101, 104, 105, 107, 100, 102, 106]
    assert vals[:, 0].tolist() == [-1, 3, 3, 4, 4, 5, 5, 5]
    docs, vals = ref.top_hits(sh, ALL, SC, [(COLUMN, 0, 1, 0, -2**63)], 4, 1)   # desc, missing last
    assert docs.tolist() == [102, 106, 101] and vals[:, 0].tolist() == [5, 5, 3]


def test_selectors():
    sh = small()
    docs, vals = ref.top_hits(sh, ALL, SC, [(COLUMN, 1, 0, 0, 100)], 8, 0)   # MIN; no value: 100
    assert docs.tolist() == [101, 103, 100, 104, 102, 105, 106, 107]
    assert vals[:, 0].tolist() == [1, 2, 4, 6, 100, 100, 100, 100]
    docs, vals = ref.top_hits(sh, ALL, SC, [(COLUMN, 1, 1, 1, -100)], 4, 0)  # MAX, descending
    assert docs.tolist() == [104, 100, 101, 103] and vals[:, 0].tolist() == [9, 8, 7, 2]


def test_docid():
    sh = small()
    docs, vals = ref.top_hits(sh, ALL, SC, [(DOCID, 0, 1, 0, 0), (COLUMN, 0, 0, 0, 0)], 3, 0)
    assert docs.tolist() == [107, 106, 105] and vals[:, 0].tolist() == [107, 106, 105]
    docs, _ = ref.top_hits(sh, ALL, SC, [(COLUMN, 2, 0, 0, 0), (DOCID, 0, 1, 0, 0)], 2, 0)
    assert docs.tolist() == [107, 106]


def test_leading_score():
    sh = small()
    docs, vals = ref.top_hits(sh, ALL, SC, [(SCORE, 0, 0, 0, 0), (COLUMN, 0, 1, 0, 0)], 8, 0)
    assert docs.tolist() == [107, 103, 100, 102, 105, 101, 104, 106]   # 3.0: missing 0 before -1; 2.0: 5, 5, missing 0; ...
    assert vals[:, 0].tolist() == SC[docs - 100].view(np.uint32).astype(np.int64).tolist()
    docs, vals = ref.top_hits(sh, ALL, SC, [(SCORE, 0, 1, 0, 0), (COLUMN, 0, 1, 0, 0)], 8, 0)
    assert docs.tolist() == [106, 101, 104, 100, 102, 105, 107, 103]
    assert np.array_equal(vals[:, 1], [5, 3, 3, 5, 5, 0, 0, -1])


def test_eight_fields():
    sh = small()
    fields = [(COLUMN, 2, 0, 0, 0), (COLUMN, 1, 0, 1, 50), (COLUMN, 0, 1, 0, 7), (COLUMN, 2, 1, 0, 0), (COLUMN, 1, 1, 0, 0),
              (COLUMN, 0, 0, 0, 0), (COLUMN, 2, 0, 0, 0), (DOCID, 0, 1, 0, 0)]
    docs, vals = ref.top_hits(sh, ALL, SC, fields, 8, 0)
    # MAX of c1 (no value: 50): 100 8 | 101 7 | 103 2 | 104 9 | others 50; ties at 50: c0 desc (missing 7), then docid desc
    assert docs.tolist() == [103, 101, 100, 104, 107, 105, 106, 102]
    assert vals.shape == (8, 8) and vals[:, 7].tolist() == docs.tolist()
