"""compile_filters (CPU): per-query kNN filter queries -> clauses, filters and filter_of. A filter only matches, so
filters equal up to their boosts share one index and the device evaluates them once."""
import numpy as np
import pytest

from nrtsearch_b200.search import BooleanQuery, BoostQuery, Occur, RangeQuery, TermQuery, compile_filters


def test_equal_filters_share_an_index_whatever_their_boosts():
    filters = [TermQuery(3), BoostQuery(TermQuery(3), 2.0), None,
               BooleanQuery().add(BoostQuery(RangeQuery(1, 2, 3), 0.5), Occur.FILTER), RangeQuery(1, 2, 3),
               BooleanQuery().add(RangeQuery(1, 2, 3), Occur.FILTER), BooleanQuery(minimum_number_should_match=1)
               .add(TermQuery(3), Occur.SHOULD)]
    carr, ncl, qarr, nf, filter_of = compile_filters(filters, len(filters))
    assert filter_of.tolist() == [0, 0, -1, 1, 2, 1, 3]
    assert nf == 4 and ncl == 4
    assert [(qarr[i].clause_begin, qarr[i].clause_end, qarr[i].min_should_match) for i in range(nf)] == \
        [(0, 1, 0), (1, 2, 0), (2, 3, 0), (3, 4, 1)]


def test_no_filters_and_length_mismatch():
    _, ncl, _, nf, filter_of = compile_filters([None, None], 2)
    assert ncl == 0 and nf == 0 and np.array_equal(filter_of, [-1, -1])
    with pytest.raises(ValueError):
        compile_filters([None], 2)
