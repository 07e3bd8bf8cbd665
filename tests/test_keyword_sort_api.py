"""The Python side of keyword sort fields that needs no GPU: SortType's nrtgpu_sort_field record, its refusals, FieldDoc value
encoding helpers, and the multi-GPU gather's refusal of a keyword Sort."""
import numpy as np
import pytest
import torch

from nrtsearch_b200 import NrtGpuUnsupported
from nrtsearch_b200.search import FieldDoc, SortType, _TermNames, _after_row, _keyword_sort_values
from nrtsearch_b200.shards import SortedPackedGather


def test_keyword_sort_field_record():
    f = SortType(3, True, True, "keyword", "middle_max").c_field()
    assert (f.kind, f.column, f.reverse, f.selector, f.missing_value) == (5, 3, 1, 3, 1)
    f = SortType(0, field_type="keyword").c_field()
    assert (f.kind, f.column, f.reverse, f.selector, f.missing_value) == (5, 0, 0, 0, 0)
    assert SortType(1, field_type="keyword", selector="middle_min").c_field().selector == 2
    with pytest.raises(ValueError):
        SortType(1, field_type="keyword", selector="median").c_field()
    for ft in ("int", "long", "float", "double"):   # MIDDLE_* stays a keyword selector
        with pytest.raises(ValueError, match="'min' or 'max'"):
            SortType(1, field_type=ft, selector="middle_min").c_field()


def test_value_encoding():
    fields = [SortType(2, field_type="keyword"), SortType(0, field_type="int")]
    terms = {(2, 0): b"a", (2, 4): "\U0001f355".encode()}
    v = np.array([[[2, 7], [10, -3], [0, 5]]], np.int64)
    looked = []
    names = _TermNames(lambda c, o: looked.append((c, o)) or terms[(c, o)])
    for _ in range(2):   # each term is looked up once
        out = _keyword_sort_values(fields, v, names)
        assert out.dtype == object and out.tolist() == [[["a", 7], ["\U0001f355", -3], [None, 5]]]
        assert all(type(x) is int for x in out[..., 1].reshape(-1))
    assert sorted(looked) == [(2, 0), (2, 4)]
    nums = np.zeros((1, 2, 1), np.int64)
    assert _keyword_sort_values([SortType(0, field_type="int")], nums, None) is nums
    seek = {(2, b"b"): 5}
    assert _after_row(fields, FieldDoc(0, values=("b", 4)), lambda c, t: seek[(c, t)]) == [5, 4]
    assert _after_row(fields, FieldDoc(0, values=(None, 4)), None) == [0, 4]
    assert _after_row(fields[:1], FieldDoc(0, 9), None) == [9]


def test_sorted_packed_gather_refuses_a_keyword_sort():
    with pytest.raises(NrtGpuUnsupported, match="keyword"):
        SortedPackedGather(2, 4, [SortType(0, field_type="int"), SortType(1, field_type="keyword")], 2, torch.device("cpu"))
    g = SortedPackedGather(2, 4, [SortType(0, field_type="int")], 2, torch.device("cpu"))   # numeric Sorts as before
    assert g.n_fields == 1
