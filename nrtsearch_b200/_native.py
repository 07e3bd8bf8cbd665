"""ctypes bindings of the in-tree native libraries.

libnrtgpu.so   -- the CUDA engine behind include/nrtgpu.h (sm_90a). There is NO fallback: if the
                  library is missing or no CUDA device is present, calls raise NrtGpuError.
libnrtsynth.so -- host-side deterministic corpus/query generators (bench + tests inputs).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))


class NrtGpuError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"nrtgpu status {status}: {message}")
        self.status = status
        self.message = message


class NrtGpuUnsupported(NrtGpuError):
    """Query shape outside the GPU path (the Java adaptor would fall through to Lucene)."""


class CollectionTimeoutException(NrtGpuError):
    """SearchCutoffWrapper.CollectionTimeoutException: the deadline passed and partial results are disallowed."""


def _load(name: str) -> C.CDLL:
    path = os.path.join(_HERE, name)
    if name == "libnrtgpu.so" and os.environ.get("NRTGPU_LIB_PATH"):   # kernel-variant experiments only
        path = os.environ["NRTGPU_LIB_PATH"]
    if not os.path.exists(path):
        raise ImportError(
            f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            f"(or `make -C nrtsearch_b200/csrc`). nrtsearch_b200 has no CPU fallback.")
    return C.CDLL(path)


i32p, i64p, f32p, u8p = (C.POINTER(t) for t in (C.c_int32, C.c_int64, C.c_float, C.c_uint8))


class ShardDesc(C.Structure):
    _fields_ = [
        ("n_docs", C.c_int32), ("doc_base", C.c_int32), ("n_terms", C.c_int32),
        ("term_off", i64p), ("post_docs", i32p), ("post_freqs", i32p),
        ("term_field", i32p), ("term_df", i64p),
        ("n_fields", C.c_int32), ("norms", C.POINTER(u8p)),
        ("field_doc_count", i64p), ("field_sum_ttf", i64p),
        ("field_k1", f32p), ("field_b", f32p),
        ("n_columns", C.c_int32), ("columns", C.POINTER(i64p)), ("column_has", C.POINTER(u8p)),
        ("live_docs", u8p),
        ("vec_dims", C.c_int32), ("vec_similarity", C.c_int32), ("vec_count", C.c_int32),
        ("vectors", C.c_void_p), ("vec_docs", i32p), ("vec_element_type", C.c_int32), ("column_offsets", C.POINTER(i64p)),
    ]


class Clause(C.Structure):
    _fields_ = [("occur", C.c_int32), ("kind", C.c_int32), ("id", C.c_int32), ("boost", C.c_float),
                ("lo", C.c_int64), ("hi", C.c_int64)]


class SearchLimits(C.Structure):
    _fields_ = [("timeout_sec", C.c_double), ("elapsed_sec", C.c_double), ("disallow_partial_results", C.c_int32),
                ("terminate_after", C.c_int32), ("terminate_after_max_recall_count", C.c_int32)]


class Sort(C.Structure):
    _fields_ = [("kind", C.c_int32), ("column", C.c_int32), ("reverse", C.c_int32), ("reserved", C.c_int32),
                ("missing_value", C.c_int64), ("after_values", C.c_void_p)]


class SortField(C.Structure):
    _fields_ = [("kind", C.c_int32), ("column", C.c_int32), ("reverse", C.c_int32), ("selector", C.c_int32),
                ("missing_value", C.c_int64)]


class Diagnostics(C.Structure):
    _fields_ = [("queue_ms", C.c_double), ("search_ms", C.c_double), ("batch_size", C.c_int32), ("reserved", C.c_int32)]


class Aggregation(C.Structure):
    _fields_ = [("kind", C.c_int32), ("column", C.c_int32), ("value_type", C.c_int32), ("size", C.c_int32),
                ("order_desc", C.c_int32), ("filter_agg", C.c_int32)]


class AggFilter(C.Structure):
    """nrtgpu_agg_filter: the filter of a FILTER aggregation, a filter query (kind 1) or a value set (kind 2)."""
    _fields_ = [("kind", C.c_int32), ("query", C.c_int32), ("column", C.c_int32), ("n_values", C.c_int32),
                ("values", C.c_void_p)]


class AggregationResult(C.Structure):
    _fields_ = [("values", C.c_void_p), ("bucket_keys", C.c_void_p), ("bucket_counts", C.c_void_p), ("n_buckets", C.c_void_p),
                ("total_buckets", C.c_void_p), ("other_counts", C.c_void_p)]


class NestedAggregation(C.Structure):
    _fields_ = [("parent", C.c_int32), ("kind", C.c_int32), ("column", C.c_int32), ("value_type", C.c_int32),
                ("top_hits", C.c_int32), ("start_hit", C.c_int32), ("orders_parent", C.c_int32), ("reserved", C.c_int32)]


class NestedSort(C.Structure):
    """nrtgpu_nested_sort: the Sort of a nested top hits, one nrtgpu_sort_order per image (orders NULL: by score), and its
    FieldDoc values output."""
    _fields_ = [("orders", C.c_void_p), ("values", C.c_void_p)]


class NestedResult(C.Structure):
    _fields_ = [("values", C.c_void_p), ("hit_docs", C.c_void_p), ("hit_scores", C.c_void_p), ("hit_counts", C.c_void_p),
                ("hit_total", C.c_void_p)]


class KeywordColumn(C.Structure):
    """nrtgpu_keyword_column: a keyword column's term dictionary and its per-doc ordinals (SORTED) or CSR of ordinals
    (SORTED_SET)."""
    _fields_ = [("n_terms", C.c_int32), ("multi_valued", C.c_int32), ("term_bytes", C.c_void_p), ("term_offsets", C.c_void_p),
                ("ords", C.c_void_p), ("doc_offsets", C.c_void_p)]


class Query(C.Structure):
    _fields_ = [("clause_begin", C.c_int32), ("clause_end", C.c_int32), ("min_should_match", C.c_int32),
                ("has_after", C.c_int32), ("after_doc", C.c_int32), ("after_score", C.c_float)]


class Node(C.Structure):
    """nrtgpu_node: a nested BooleanQuery (kind 0), DisjunctionMaxQuery (kind 1), ConstantScoreQuery (kind 3),
    MinScoreQuery (kind 4) or NestedQuery (kind 6, a block join whose score mode is min_should_match) of a query tree;
    boost is that of kinds 3 and 4, min_score that of kind 4."""
    _fields_ = [("kind", C.c_int32), ("clause_begin", C.c_int32), ("clause_end", C.c_int32), ("min_should_match", C.c_int32),
                ("tie_breaker", C.c_float), ("boost", C.c_float), ("min_score", C.c_float)]


class Phrase(C.Structure):
    """nrtgpu_phrase: a PhraseQuery leaf (clause kind 4) or a MultiPhraseQuery leaf (clause kind 6, NRTGPU_MULTI_PHRASE:
    terms that share a position are alternatives) of a query tree, its terms phrase_terms[term_begin:term_end]."""
    _fields_ = [("term_begin", C.c_int32), ("term_end", C.c_int32), ("slop", C.c_int32), ("reserved", C.c_int32)]


class PhraseTerm(C.Structure):
    """nrtgpu_phrase_term: a term of a phrase and its PhraseQuery / MultiPhraseQuery position."""
    _fields_ = [("term", C.c_int32), ("position", C.c_int32)]


# every symbol include/nrtgpu.h declares (tests/test_abi.py checks the header against this list)
NRTGPU_SYMBOLS = [
    "nrtgpu_last_error", "nrtgpu_version", "nrtgpu_init", "nrtgpu_shutdown", "nrtgpu_index_build",
    "nrtgpu_index_close", "nrtgpu_index_device_bytes", "nrtgpu_search_bool", "nrtgpu_batch_prepare",
    "nrtgpu_batch_run", "nrtgpu_batch_fetch", "nrtgpu_batch_device_results", "nrtgpu_batch_stats",
    "nrtgpu_batch_stage_ms", "nrtgpu_batch_reset_timing", "nrtgpu_batch_bind_output", "nrtgpu_batch_free", "nrtgpu_search_knn", "nrtgpu_search_knn_timed", "nrtgpu_merge_topk_device",
    "nrtgpu_blend_rrf", "nrtgpu_blend_scores", "nrtgpu_rescore_combine", "nrtgpu_knn_last_uncertified", "nrtgpu_packed_words", "nrtgpu_search_sorted", "nrtgpu_search_bool_aggs", "nrtgpu_score_docs", "nrtgpu_rescore_query", "nrtgpu_fetch_columns", "nrtgpu_index_set_live_docs", "nrtgpu_index_update_stats", "nrtgpu_searcher_create", "nrtgpu_searcher_search_bool", "nrtgpu_searcher_close", "nrtgpu_batcher_create", "nrtgpu_batcher_submit", "nrtgpu_batcher_stats", "nrtgpu_batcher_close", "nrtgpu_search_bool_ex", "nrtgpu_search_bool_packed", "nrtgpu_batch_set_limits", "nrtgpu_batch_fetch_ex", "nrtgpu_batch_bind_packed", "nrtgpu_merge_topk_packed",
    "nrtgpu_search_knn_filtered", "nrtgpu_knn_filter_stats",
    "nrtgpu_sort_order_create", "nrtgpu_sort_order_device_bytes", "nrtgpu_sort_order_close", "nrtgpu_search_sorted_fields",
    "nrtgpu_search_tree", "nrtgpu_batch_prepare_tree",
    "nrtgpu_index_add_positions", "nrtgpu_index_add_parents", "nrtgpu_search_tree_phrases", "nrtgpu_batch_prepare_tree_phrases",
    "nrtgpu_score_docs_tree", "nrtgpu_rescore_query_tree",
    "nrtgpu_search_bool_aggs_nested",
    "nrtgpu_sorted_packed_words", "nrtgpu_search_sorted_fields_packed", "nrtgpu_merge_sorted_packed",
    "nrtgpu_searcher_search_sorted_fields", "nrtgpu_searcher_search_tree_phrases", "nrtgpu_searcher_search_knn",
    "nrtgpu_searcher_search_knn_filtered", "nrtgpu_searcher_search_bool_aggs_nested",
    "nrtgpu_search_bool_aggs_filtered", "nrtgpu_searcher_search_bool_aggs_filtered",
    "nrtgpu_search_bool_aggs_sorted_hits", "nrtgpu_searcher_search_bool_aggs_sorted_hits",
    "nrtgpu_search_tree_aggs", "nrtgpu_searcher_search_tree_aggs",
    "nrtgpu_index_add_keyword_columns", "nrtgpu_index_keyword_term", "nrtgpu_searcher_keyword_term",
    "nrtgpu_index_keyword_seek", "nrtgpu_searcher_keyword_seek",
    "nrtgpu_index_keyword_range", "nrtgpu_searcher_keyword_range",
]

_gpu = None
_synth = None


def gpu_lib() -> C.CDLL:
    global _gpu
    if _gpu is None:
        lib = _load("libnrtgpu.so")
        lib.nrtgpu_last_error.restype = C.c_char_p
        lib.nrtgpu_index_device_bytes.restype = C.c_int64
        lib.nrtgpu_index_device_bytes.argtypes = [C.c_void_p]
        lib.nrtgpu_init.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        lib.nrtgpu_shutdown.argtypes = [C.c_void_p]
        lib.nrtgpu_shutdown.restype = None
        lib.nrtgpu_index_build.argtypes = [C.c_void_p, C.POINTER(ShardDesc), C.POINTER(C.c_void_p)]
        lib.nrtgpu_index_close.argtypes = [C.c_void_p]
        lib.nrtgpu_search_bool.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32,
                                           C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_batch_prepare.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32,
                                             C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        lib.nrtgpu_batch_run.argtypes = [C.c_void_p, C.c_void_p]
        lib.nrtgpu_batch_fetch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p]
        lib.nrtgpu_batch_device_results.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                                    C.POINTER(C.c_void_p)]
        lib.nrtgpu_batch_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int32),
                                           C.POINTER(C.c_int64)]
        lib.nrtgpu_batch_stage_ms.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_float)]
        lib.nrtgpu_batch_reset_timing.argtypes = [C.c_void_p]
        lib.nrtgpu_batch_bind_output.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_batch_free.argtypes = [C.c_void_p]
        lib.nrtgpu_search_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_search_knn_timed.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p]
        lib.nrtgpu_search_bool_ex.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32,
                                              C.c_int32, C.c_int32, C.POINTER(SearchLimits), C.c_void_p] + [C.c_void_p] * 7
        lib.nrtgpu_search_tree.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Node), C.c_int32, C.POINTER(Query),
                                           C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(SearchLimits), C.c_void_p] + \
                                          [C.c_void_p] * 7
        lib.nrtgpu_batch_prepare_tree.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Node), C.c_int32,
                                                  C.POINTER(Query), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                  C.POINTER(C.c_void_p)]
        lib.nrtgpu_index_add_positions.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        lib.nrtgpu_index_add_parents.argtypes = [C.c_void_p, C.c_int32]
        lib.nrtgpu_index_add_keyword_columns.argtypes = [C.c_void_p, C.POINTER(KeywordColumn), C.c_int32]
        lib.nrtgpu_index_keyword_term.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
        lib.nrtgpu_searcher_keyword_term.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32),
                                                     C.POINTER(C.c_int32)]
        lib.nrtgpu_index_keyword_seek.argtypes = [C.c_void_p, C.c_int32, C.c_char_p, C.c_int32, C.POINTER(C.c_int64)]
        lib.nrtgpu_searcher_keyword_seek.argtypes = [C.c_void_p, C.c_int32, C.c_char_p, C.c_int32, C.POINTER(C.c_int64)]
        for fn in (lib.nrtgpu_index_keyword_range, lib.nrtgpu_searcher_keyword_range):
            fn.argtypes = [C.c_void_p, C.c_int32, C.c_char_p, C.c_int32, C.c_char_p, C.c_int32, C.c_int32, C.POINTER(C.c_int64),
                           C.POINTER(C.c_int64)]
        lib.nrtgpu_search_tree_phrases.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Node), C.c_int32,
                                                   C.POINTER(Phrase), C.c_int32, C.POINTER(PhraseTerm), C.c_int32, C.POINTER(Query),
                                                   C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(SearchLimits), C.c_void_p] + \
                                                  [C.c_void_p] * 7
        lib.nrtgpu_batch_prepare_tree_phrases.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Node), C.c_int32,
                                                          C.POINTER(Phrase), C.c_int32, C.POINTER(PhraseTerm), C.c_int32,
                                                          C.POINTER(Query), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                          C.POINTER(C.c_void_p)]
        lib.nrtgpu_search_bool_packed.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32,
                                                  C.c_int32, C.c_int32, C.POINTER(SearchLimits), C.c_void_p, C.c_void_p]
        lib.nrtgpu_search_sorted.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32,
                                             C.c_int32, C.POINTER(Sort), C.POINTER(SearchLimits), C.c_void_p] + [C.c_void_p] * 7
        lib.nrtgpu_sort_order_create.argtypes = [C.c_void_p, C.POINTER(SortField), C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]
        lib.nrtgpu_sort_order_device_bytes.argtypes = [C.c_void_p]
        lib.nrtgpu_sort_order_device_bytes.restype = C.c_int64
        lib.nrtgpu_sort_order_close.argtypes = [C.c_void_p]
        lib.nrtgpu_search_sorted_fields.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32,
                                                    C.c_int32, C.c_int32, C.c_void_p, C.POINTER(SearchLimits), C.c_void_p] + [C.c_void_p] * 7
        lib.nrtgpu_search_bool_aggs.argtypes =[C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32, C.c_int32,
                                                C.POINTER(Aggregation), C.c_int32, C.POINTER(AggregationResult), C.c_void_p] + [C.c_void_p] * 4
        lib.nrtgpu_search_bool_aggs_nested.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32,
                                                       C.c_int32, C.POINTER(Aggregation), C.c_int32, C.POINTER(AggregationResult),
                                                       C.POINTER(NestedAggregation), C.c_int32, C.POINTER(NestedResult),
                                                       C.c_void_p] + [C.c_void_p] * 4
        lib.nrtgpu_score_docs.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_rescore_query.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32, C.c_void_p,
                                             C.c_int32, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_score_docs_tree.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Node), C.c_int32, C.POINTER(Phrase),
                                               C.c_int32, C.POINTER(PhraseTerm), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_rescore_query_tree.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Node), C.c_int32,
                                                  C.POINTER(Phrase), C.c_int32, C.POINTER(PhraseTerm), C.c_int32, C.POINTER(Query),
                                                  C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_fetch_columns.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_index_set_live_docs.argtypes = [C.c_void_p, C.c_void_p]
        lib.nrtgpu_index_update_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_searcher_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.POINTER(C.c_void_p)]
        lib.nrtgpu_searcher_search_bool.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_int32, C.c_int32,
                                                    C.c_int32, C.POINTER(SearchLimits), C.c_void_p] + [C.c_void_p] * 5
        lib.nrtgpu_searcher_close.argtypes = [C.c_void_p]
        lib.nrtgpu_sorted_packed_words.argtypes = [C.c_int32, C.c_int32, C.c_int32]
        lib.nrtgpu_sorted_packed_words.restype = C.c_int64
        lib.nrtgpu_search_sorted_fields_packed.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Query),
                                                           C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.POINTER(SearchLimits),
                                                           C.c_void_p, C.c_void_p]
        lib.nrtgpu_merge_sorted_packed.argtypes = [C.c_void_p, C.POINTER(SortField), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                   C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_searcher_search_sorted_fields.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.POINTER(Clause), C.c_int32,
                                                             C.POINTER(Query), C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                                             C.POINTER(SearchLimits), C.c_void_p] + [C.c_void_p] * 7
        lib.nrtgpu_searcher_search_tree_phrases.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Node), C.c_int32,
                                                            C.POINTER(Phrase), C.c_int32, C.POINTER(PhraseTerm), C.c_int32,
                                                            C.POINTER(Query), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                            C.POINTER(SearchLimits), C.c_void_p] + [C.c_void_p] * 7
        lib.nrtgpu_searcher_search_knn.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_searcher_search_knn_filtered.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.POINTER(Clause),
                                                            C.c_int32, C.POINTER(Query), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                            C.c_void_p, C.c_void_p]
        lib.nrtgpu_searcher_search_bool_aggs_nested.argtypes = lib.nrtgpu_search_bool_aggs_nested.argtypes
        lib.nrtgpu_search_bool_aggs_filtered.argtypes = lib.nrtgpu_search_bool_aggs_nested.argtypes[:13] + \
            [C.POINTER(AggFilter), C.POINTER(Clause), C.c_int32, C.POINTER(Query), C.c_int32, C.c_void_p] + [C.c_void_p] * 4
        lib.nrtgpu_searcher_search_bool_aggs_filtered.argtypes = lib.nrtgpu_search_bool_aggs_filtered.argtypes
        lib.nrtgpu_search_bool_aggs_sorted_hits.argtypes = lib.nrtgpu_search_bool_aggs_filtered.argtypes[:13] + \
            [C.POINTER(NestedSort)] + lib.nrtgpu_search_bool_aggs_filtered.argtypes[13:]
        lib.nrtgpu_searcher_search_bool_aggs_sorted_hits.argtypes = lib.nrtgpu_search_bool_aggs_sorted_hits.argtypes
        # the tree and phrase arguments of nrtgpu_search_tree_phrases, then those of nrtgpu_search_bool_aggs_sorted_hits
        lib.nrtgpu_search_tree_aggs.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.POINTER(Node), C.c_int32, C.POINTER(Phrase),
                                                C.c_int32, C.POINTER(PhraseTerm), C.c_int32] + \
            lib.nrtgpu_search_bool_aggs_sorted_hits.argtypes[3:]
        lib.nrtgpu_searcher_search_tree_aggs.argtypes = lib.nrtgpu_search_tree_aggs.argtypes
        lib.nrtgpu_batcher_create.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        lib.nrtgpu_batcher_submit.argtypes = [C.c_void_p, C.POINTER(Clause), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(Diagnostics)]
        lib.nrtgpu_batcher_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        lib.nrtgpu_batcher_close.argtypes = [C.c_void_p]
        lib.nrtgpu_batch_set_limits.argtypes = [C.c_void_p, C.POINTER(SearchLimits)]
        lib.nrtgpu_batch_fetch_ex.argtypes = [C.c_void_p] * 9
        lib.nrtgpu_packed_words.argtypes = [C.c_int32, C.c_int32]
        lib.nrtgpu_packed_words.restype = C.c_int64
        lib.nrtgpu_batch_bind_packed.argtypes = [C.c_void_p, C.c_void_p]
        lib.nrtgpu_merge_topk_packed.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_knn_last_uncertified.argtypes = [C.c_void_p]
        lib.nrtgpu_knn_last_uncertified.restype = C.c_int32
        lib.nrtgpu_search_knn_filtered.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.POINTER(Clause),
                                                   C.c_int32, C.POINTER(Query), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_void_p, C.c_void_p]
        lib.nrtgpu_knn_filter_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        lib.nrtgpu_merge_topk_device.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 7
        lib.nrtgpu_blend_rrf.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
        lib.nrtgpu_blend_scores.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtgpu_rescore_combine.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_double, C.c_double]
        _gpu = lib
    return _gpu


def check(rc: int) -> None:
    if rc != 0:
        msg = gpu_lib().nrtgpu_last_error().decode("utf-8", "replace")
        raise (NrtGpuUnsupported if rc == 3 else CollectionTimeoutException if rc == 5 else NrtGpuError)(rc, msg)


def synth_lib() -> C.CDLL:
    global _synth
    if _synth is None:
        lib = _load("libnrtsynth.so")
        lib.nrtsynth_corpus_begin.restype = C.c_void_p
        lib.nrtsynth_corpus_begin.argtypes = [C.c_int64, C.c_int64, C.c_int, C.c_uint64, C.c_int, C.c_double, C.c_double,
                                              C.c_void_p, C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        lib.nrtsynth_corpus_fill.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.nrtsynth_corpus_fill.restype = None
        lib.nrtsynth_corpus_end.argtypes = [C.c_void_p]
        lib.nrtsynth_corpus_end.restype = None
        lib.nrtsynth_int_column.argtypes = [C.c_int64, C.c_int64, C.c_uint64, C.c_int32, C.c_void_p]
        lib.nrtsynth_int_column.restype = None
        lib.nrtsynth_queries.argtypes = [C.c_int, C.c_int, C.c_uint64, C.c_double, C.c_double, C.c_int, C.c_void_p]
        lib.nrtsynth_queries.restype = None
        lib.nrtsynth_uniform.argtypes = [C.c_int64, C.c_uint64, C.c_void_p]
        lib.nrtsynth_uniform.restype = None
        lib.nrtsynth_normal_f32.argtypes = [C.c_int64, C.c_int64, C.c_uint64, C.c_void_p]
        lib.nrtsynth_normal_f32.restype = None
        _synth = lib
    return _synth
