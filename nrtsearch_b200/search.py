"""Host-side mirror of the reference's query-execution interface for the hot path.

Names and argument meaning follow the Lucene/nrtsearch API at the three call sites the engine replaces
(SURVEY.md 8b) so parity tests read like the reference's own:

  IndexSearcher.search(Query, CollectorManager)   src/main/java/com/yelp/nrtsearch/server/handler/SearchHandler.java:1412
  BooleanQuery / TermQuery / RangeQuery / BoostQuery / MatchAllDocsQuery
                                                  src/main/java/com/yelp/nrtsearch/server/query/QueryNodeMapper.java:257-283
  RelevanceCollector (numHitsToCollect, totalHitsThreshold, searchAfter)
                                                  src/main/java/com/yelp/nrtsearch/server/search/collectors/RelevanceCollector.java:42-69
  KnnQuery / ExactVectorQuery                     src/main/java/com/yelp/nrtsearch/server/search/KnnUtils.java:47-66

All execution happens in libnrtgpu.so (CUDA); this module only marshals.
"""
from __future__ import annotations

import ctypes as C
import enum
import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _native
from ._native import (AggFilter as CAggFilter, Aggregation as CAgg, AggregationResult as CAggResult, NestedAggregation as CNested,
                      NestedSort as CNestedSort,
                      NestedResult as CNestedResult, Clause, CollectionTimeoutException, NrtGpuError,
                      NrtGpuUnsupported, Query as CQuery, SearchLimits, Sort as CSort, check)
from .index import HostShard, PinnedDesc

TOTAL_HITS_THRESHOLD = 1000  # SearchRequestProcessor.TOTAL_HITS_THRESHOLD (:102)
INT_MAX = 2**31 - 1


class Occur(enum.IntEnum):
    SHOULD = 0
    MUST = 1
    FILTER = 2
    MUST_NOT = 3


@dataclass(frozen=True)
class TermQuery:
    term: int  # the adaptor's dense (field, term) id


@dataclass(frozen=True)
class RangeQuery:
    """IndexOrDocValuesQuery(PointRangeQuery, SortedNumericDocValuesRangeQuery): inclusive bounds in the
    sortable-long domain (IntFieldDef.getRangeQuery :124-158 folds exclusive bounds with +-1)."""
    column: int
    lower: int = -(2**63)
    upper: int = 2**63 - 1


@dataclass(frozen=True)
class KeywordRangeQuery:
    """TermRangeQuery on an atom field (AtomFieldDef.getRangeQuery; SortedSetDocValuesField.newSlowRangeQuery on a field
    with doc values only): keyword column `column` (HostShard.keyword_columns) has a term in the range, in unsigned-byte
    order. lower / upper: str (UTF-8) or bytes, already normalized as the field indexes its terms, or None for an open
    end. Constant-score: a matching doc scores the boost, as RangeQuery does. Usable wherever RangeQuery is; each searcher
    turns it into a code range of its dictionary (keyword_range)."""
    column: int
    lower: object = None
    upper: object = None
    include_lower: bool = True
    include_upper: bool = True


@dataclass(frozen=True)
class KeywordPrefixQuery:
    """PrefixQuery on an atom field (AtomFieldDef.getPrefixQuery) with a constant-score rewrite: keyword column `column`
    has a term starting with `prefix` (str or bytes). Usable wherever RangeQuery is, as KeywordRangeQuery."""
    column: int
    prefix: object = b""


@dataclass(frozen=True)
class _KeywordCodes:
    """a KeywordRangeQuery / KeywordPrefixQuery resolved by a searcher: the inclusive code range [lo, hi] of keyword column
    `column` in its dictionary (an NRTGPU_KEYWORD_RANGE clause)"""
    column: int
    lo: int
    hi: int


@dataclass(frozen=True)
class MatchAllDocsQuery:
    pass


@dataclass(frozen=True)
class BoostQuery:
    query: object
    boost: float


@dataclass
class DisjunctionMaxQuery:
    """DisjunctionMaxQuery(disjuncts, tieBreakerMultiplier): what multi_match BEST_FIELDS maps to (QueryNodeMapper.java:429-497).
    A doc matches if any disjunct does and scores max + tie_breaker * (the other matching disjuncts' scores)."""
    disjuncts: List[object] = field(default_factory=list)
    tie_breaker: float = 0.0


@dataclass(frozen=True)
class ConstantScoreQuery:
    """ConstantScoreQuery(filter) (QueryNodeMapper.java:194, :635-640): a doc matches when `filter` does and scores the
    product of the BoostQuerys around this query (1 without them); nothing inside it scores. ExistsQuery(field) is one
    over the _field_names term of the field (INTEGRATION.md). A node of a query tree (GpuIndexSearcher.search_tree)."""
    filter: object


@dataclass(frozen=True)
class MinScoreQuery:
    """MinScoreQuery(query, min_score), built by the reference as MinThresholdQuery (QueryNodeMapper.java:199, :642-656):
    a doc matches when `query` does with a float score s >= min_score, and scores s times the product of the BoostQuerys
    around this query; `query` is scored with boost 1 (its own BoostQuerys still apply), even where the tree only
    filters. min_score < 0 is refused; 0 returns `query` itself with the outer boosts folded into it, as the reference
    does; NaN matches nothing. A node of a query tree (GpuIndexSearcher.search_tree)."""
    query: object
    min_score: float


_NESTED_SCORE_MODES = {"none": 0, "avg": 1, "max": 2, "min": 3, "sum": 4}


@dataclass(frozen=True)
class NestedQuery:
    """NestedQuery(query, path_term, score_mode) (QueryNodeMapper.getNestedQuery): a block join. `query` runs over the
    child docs of the nested path whose _nested_path term is `path_term` (the adaptor's term id), without live docs; each
    parent doc (HostShard.parent_term, the _nested_path:_root term) that follows matching children matches and scores
    the fold of their scores: "none" 0, "sum" the double sum in child order, "avg" that sum / n, "max" / "min" the largest /
    smallest. BoostQuerys around it fold into `query`'s leaves. A node of a query tree (GpuIndexSearcher.search_tree)
    whose child query is BooleanQuery{FILTER TermQuery(path_term), MUST query}, as the reference builds it."""
    query: object
    path_term: int
    score_mode: str = "none"

    def mode(self) -> int:
        if self.score_mode not in _NESTED_SCORE_MODES:
            raise ValueError(f"NestedQuery: unknown score_mode {self.score_mode!r}")
        return _NESTED_SCORE_MODES[self.score_mode]

    def child_query(self) -> "BooleanQuery":
        return BooleanQuery().add(TermQuery(int(self.path_term)), Occur.FILTER).add(self.query, Occur.MUST)


@dataclass
class PhraseQuery:
    """PhraseQuery(slop, terms, positions): what match_phrase maps to (QueryNodeMapper.java:285-291, :397-427). All terms on
    one text field; positions default to 0, 1, 2, ... as PhraseQuery.Builder.add(term) assigns them. Runs on the window
    engine as a leaf of a query tree (GpuIndexSearcher.search_tree) over an image with positions."""
    terms: List[int] = field(default_factory=list)   # the adaptor's dense (field, term) ids
    positions: Optional[List[int]] = None
    slop: int = 0

    def term_positions(self) -> List[Tuple[int, int]]:
        pos = list(range(len(self.terms))) if self.positions is None else list(self.positions)
        if len(pos) != len(self.terms):
            raise ValueError("PhraseQuery: one position per term")
        return [(int(t), int(p)) for t, p in zip(self.terms, pos)]


@dataclass
class MultiPhraseQuery:
    """MultiPhraseQuery(terms, positions, slop): a phrase whose position i holds any of the alternative terms terms[i]
    (match_phrase over stacked synonyms; the query MatchPhrasePrefixQuery rewrites to). All terms on one text field, term
    ids as for PhraseQuery; positions default to 0, 1, 2, ... and must ascend. A doc matches position i when any of
    terms[i] occurs there; one position is the BooleanQuery of SHOULD TermQuerys over its alternatives, no position (or an
    empty one) matches nothing. Runs on the window engine as a leaf of a query tree (GpuIndexSearcher.search_tree), the
    alternatives of a position merged on the device (nrtgpu.h NRTGPU_MULTI_PHRASE)."""
    terms: List[List[int]] = field(default_factory=list)
    positions: Optional[List[int]] = None
    slop: int = 0

    def term_positions(self) -> List[Tuple[int, int]]:
        """(term, position) of every alternative, position after position; [] when the query matches nothing"""
        pos = list(range(len(self.terms))) if self.positions is None else [int(p) for p in self.positions]
        if len(pos) != len(self.terms):
            raise ValueError("MultiPhraseQuery: one position per term array")
        if len(set(pos)) != len(pos):
            raise ValueError("MultiPhraseQuery: one term array per position")
        if any(len(alts) == 0 for alts in self.terms):
            return []
        return [(int(t), p) for alts, p in zip(self.terms, pos) for t in alts]


@dataclass
class MatchPhrasePrefixQuery:
    """match_phrase_prefix (reference MatchPhrasePrefixQuery.java): terms[i] are the analyzed tokens at position i (several
    at one position: stacked synonyms) and `expansions` the indexed terms the last token's prefix expands to, which the
    adaptor finds in the term dictionary (at most max_expansions, default 50; INTEGRATION.md). It rewrites as the
    reference does: no expansion matches nothing; otherwise a MultiPhraseQuery of terms followed by the expansions, so a
    one-token query is the disjunction of its expansions. Term ids as for PhraseQuery."""
    terms: List[List[int]] = field(default_factory=list)
    expansions: List[int] = field(default_factory=list)
    slop: int = 0

    def rewrite(self) -> MultiPhraseQuery:
        if not self.expansions:
            return MultiPhraseQuery([], None, int(self.slop))
        return MultiPhraseQuery([list(t) for t in self.terms] + [list(self.expansions)], None, int(self.slop))


@dataclass(frozen=True)
class BooleanClause:
    query: object
    occur: Occur


@dataclass
class BooleanQuery:
    clauses: List[BooleanClause] = field(default_factory=list)
    minimum_number_should_match: int = 0

    def add(self, query, occur: Occur) -> "BooleanQuery":
        self.clauses.append(BooleanClause(query, Occur(occur)))
        return self


def boolean_query_from_proto(clauses: Sequence[Tuple[object, Occur]], minimum_number_should_match: int = 0) -> BooleanQuery:
    """QueryNodeMapper.getBooleanQuery (:257-283): empty => MatchAllDocs MUST; all MUST_NOT => add MatchAllDocs FILTER."""
    bq = BooleanQuery(minimum_number_should_match=minimum_number_should_match)
    if not clauses:
        return bq.add(MatchAllDocsQuery(), Occur.MUST)
    all_must_not = True
    for q, occ in clauses:
        bq.add(q, occ)
        if occ != Occur.MUST_NOT:
            all_must_not = False
    if all_must_not:
        bq.add(MatchAllDocsQuery(), Occur.FILTER)
    return bq


@dataclass
class ScoreDoc:
    doc: int
    score: float


class Relation(enum.IntEnum):
    EQUAL_TO = 0
    GREATER_THAN_OR_EQUAL_TO = 1


@dataclass
class TotalHits:
    value: int
    relation: Relation


@dataclass
class TopDocs:
    total_hits: TotalHits
    score_docs: List[ScoreDoc]


@dataclass
class RelevanceCollector:
    """DocCollector config (CollectorCreatorContext.java:36-53, DocCollector.java wrappers): numHitsToCollect,
    totalHitsThreshold, searchAfter; timeoutSec / disallowPartialResults (SearchCutoffWrapper.java:164-202);
    terminateAfter / terminateAfterMaxRecallCount (TerminateAfterWrapper.java:85-162)."""
    num_hits_to_collect: int
    total_hits_threshold: int = TOTAL_HITS_THRESHOLD
    search_after: Optional[ScoreDoc] = None
    timeout_sec: float = 0.0
    elapsed_sec: float = 0.0
    disallow_partial_results: bool = False
    terminate_after: int = 0
    terminate_after_max_recall_count: int = 0

    def limits(self) -> Optional[SearchLimits]:
        if self.timeout_sec <= 0 and self.terminate_after <= 0:
            return None
        return SearchLimits(self.timeout_sec, self.elapsed_sec, 1 if self.disallow_partial_results else 0,
                            self.terminate_after, self.terminate_after_max_recall_count)


def float_to_sortable_int(f: float) -> int:
    """NumericUtils.floatToSortableInt: the order-preserving int of a float (how FloatFieldDef stores doc values)."""
    b = int(np.float32(f).view(np.int32))
    return b ^ ((b >> 31) & 0x7fffffff)


def double_to_sortable_long(d: float) -> int:
    """NumericUtils.doubleToSortableLong."""
    b = int(np.float64(d).view(np.int64))
    return b ^ ((b >> 63) & 0x7fffffffffffffff)


@dataclass(frozen=True)
class SortType:
    """SortType of the search request for ONE sort field (SortParser.parseSort :54-95): a numeric doc-value column,
    "docid" or "score" (higher scores first unless reverse). field_type picks the missing value exactly as the reference's
    FieldDefs do (IntFieldDef.java:103, LongFieldDef.java:103, FloatFieldDef.java:105, DoubleFieldDef.java:105): MAX /
    +Infinity when missing_last, else MIN / -Infinity -- irrespective of reverse. selector: which value of a multi-valued
    column sorts the doc, "min" (the default) or "max" (NumberFieldDef.java:266-278, SortedNumericSelector).
    field_type "keyword": field is a keyword column of the shard (HostShard.keyword_columns), sorted by its term in
    unsigned-byte order (AtomFieldDef.getSortField: SortField STRING, or SortedSetSortField on a multi-valued column,
    whose selector may also be "middle_min" or "middle_max"); a doc without a value sorts first, or last when missing_last,
    and reverse reverses the whole order, the missing position included. Its FieldDoc values are str, or None for no
    value."""
    field: object            # column id, "docid" or "score"
    reverse: bool = False
    missing_last: bool = False
    field_type: str = "long"   # int | long | float | double | keyword
    selector: str = "min"

    @property
    def keyword(self) -> bool:
        return self.field_type == "keyword" and self.field not in ("docid", "score")

    def missing_value(self) -> int:
        if self.field in ("docid", "score"):
            return 0
        hi = self.missing_last
        if self.field_type == "keyword":   # STRING_FIRST 0 / STRING_LAST 1
            return 1 if hi else 0
        if self.field_type == "int":
            return 2**31 - 1 if hi else -(2**31)
        if self.field_type == "long":
            return 2**63 - 1 if hi else -(2**63)
        if self.field_type == "float":
            return float_to_sortable_int(float("inf") if hi else float("-inf"))
        if self.field_type == "double":
            return double_to_sortable_long(float("inf") if hi else float("-inf"))
        raise ValueError(f"field type {self.field_type} does not support sorting")

    def c_field(self) -> _native.SortField:
        if self.keyword:
            if self.selector not in _SELECTORS:
                raise ValueError(f"selector must be one of {', '.join(map(repr, _SELECTORS))}, not {self.selector!r}")
            return _native.SortField(5, int(self.field), 1 if self.reverse else 0, _SELECTORS.index(self.selector),
                                     self.missing_value())
        if self.selector not in ("min", "max"):
            raise ValueError(f"selector must be 'min' or 'max', not {self.selector!r}")
        kind = 3 if self.field == "score" else 2 if self.field == "docid" else 1
        return _native.SortField(kind, int(self.field) if kind == 1 else 0, 1 if self.reverse else 0,
                                 1 if self.selector == "max" else 0, self.missing_value())


_SELECTORS = ("min", "max", "middle_min", "middle_max")   # NRTGPU_SELECT_*: SortedSetSelector.Type of a keyword sort


def _keyword_sort_values(fields: Sequence[SortType], values: np.ndarray, names) -> np.ndarray:
    """FieldDoc values [..., n_fields] of a Sort; with a keyword field, an object array whose keyword entries are str
    (code 2i + 2: term i, through names(column, ords), a _TermNames) or None (code 0: no value) and whose other entries are
    int; an all-numeric Sort's int64 array unchanged"""
    kw = [j for j, f in enumerate(fields) if isinstance(f, SortType) and f.keyword]
    if not kw:
        return values
    out = np.empty(values.shape, object)   # (None everywhere)
    for j, f in enumerate(fields):
        codes, col = values[..., j], out[..., j]   # (col: a view of out)
        if j not in kw:
            col[...] = codes
            continue
        held = codes != 0
        col[held] = names(int(f.field), codes[held] // 2 - 1)
    return out


class _TermNames:
    """The str of keyword terms by ordinal, per column, each looked up and decoded once (term(column, ord) -> bytes): a
    page's keyword values become str by one indexing of the column's array, whatever its number of distinct terms."""

    def __init__(self, term):
        self.term, self.cols = term, {}

    def __call__(self, column: int, ords: np.ndarray) -> np.ndarray:
        ords = np.asarray(ords, np.int64)
        names, have = self.cols.get(column, (np.empty(0, object), np.zeros(0, bool)))
        hi = int(ords.max()) + 1 if len(ords) else 0
        if hi > len(names):
            m = max(hi, 2 * len(names))
            names = np.concatenate([names, np.empty(m - len(names), object)])
            have = np.concatenate([have, np.zeros(m - len(have), bool)])
            self.cols[column] = (names, have)
        for o in np.unique(ords[~have[ords]]):
            names[o] = self.term(column, int(o)).decode("utf-8")
            have[o] = True
        return names[ords]


def _after_row(fields: Sequence[SortType], a: "FieldDoc", seek) -> list:
    """the int64 after values of FieldDoc a: a keyword field's str (or bytes) becomes its code through seek(column, bytes),
    None the null code 0; an int is taken as a code already"""
    vals = list(a.values) if a.values is not None else [a.value]
    for j, f in enumerate(fields[:len(vals)]):
        if isinstance(f, SortType) and f.keyword:
            v = vals[j]
            vals[j] = 0 if v is None else int(v) if isinstance(v, (int, np.integer)) else seek(int(f.field), _utf8_bytes(v))
    return vals


def _utf8_bytes(v) -> bytes:
    return v.encode("utf-8") if isinstance(v, str) else bytes(v)


def _seek(fn, *args) -> int:
    """the sort code of one keyword term through nrtgpu_index_keyword_seek / nrtgpu_searcher_keyword_seek (fn bound to
    its handle and column, args ending with the term's bytes)"""
    code = C.c_int64()
    t = args[-1]
    check(fn(*args[:-1], t, len(t), C.byref(code)))
    return int(code.value)


@dataclass
class SortFieldCollector:
    """SortFieldCollector.java:44-105: numHitsToCollect + the query's Sort (one SortType, or a sequence of up to 8);
    searchAfter is a FieldDoc (value, doc), or (values, doc) for a sequence."""
    num_hits_to_collect: int
    sort: object = None
    timeout_sec: float = 0.0
    terminate_after: int = 0


@dataclass(frozen=True)
class TermsCollector:
    """TermsCollector over a numeric doc-value field ({Int,Long,Float,Double}TermsCollectorManager): `size` buckets ordered
    by count (BucketOrder COUNT, desc by default). field_type "keyword": column is a keyword column of the shard
    (HostShard.keyword_columns, OrdinalTermsCollectorManager), a doc of a multi-valued one counts once per term, and the
    result's "keys" is an object array of str (None past a query's "n"). nested: up to 4 (name, MinCollector | MaxCollector | SumCollector |
    TopHitsCollector) computed per bucket (Collector.nestedCollectors); order_by: the name of a nested min / max / sum
    that orders the buckets instead of the count (BucketOrder by a nested collector, in the order_desc direction)."""
    column: int
    size: int
    order_desc: bool = True
    field_type: str = "long"
    nested: tuple = ()
    order_by: Optional[str] = None


@dataclass(frozen=True)
class TopHitsCollector:
    """TopHitsCollector (TopHitsCollectorManager): a bucket's hits by score descending, then doc ascending, positions
    [start_hit, top_hits). sort (querySort): a SortType or a sequence of up to 8, as SortFieldCollector.sort; the hits are
    then in that Sort's order, ties by doc, their scores NaN, and the result gains "sort_values" (FieldDoc.fields of every
    hit). Nested in a terms or filter collector it works per bucket; in `additional` (top level) it sees every doc the
    query collects: its result is {"docs", "scores" [nq, top_hits - start_hit], "counts", "total_hits" [nq] (the query's
    exact totalHits)[, "sort_values" [nq, top_hits - start_hit, n_fields]]}."""
    top_hits: int
    start_hit: int = 0
    sort: object = None

    def sort_fields(self) -> List[SortType]:
        return [self.sort] if isinstance(self.sort, SortType) else list(self.sort)


@dataclass(frozen=True)
class MinCollector:
    column: int
    field_type: str = "long"


@dataclass(frozen=True)
class MaxCollector:
    column: int
    field_type: str = "long"


@dataclass(frozen=True)
class SumCollector:
    column: int
    field_type: str = "long"


@dataclass(frozen=True)
class ValueSetFilter:
    """The set filter of a FilterCollector (FilterCollectorManager.SetQueryFilter over a TermInSetQuery): a doc passes when one
    of its values of `column` (single- or multi-valued) is in `values`, numbers of the field's type compared as Java's boxed
    equals does, by their bits (-0.0 != 0.0, NaN == NaN). A set of another term type than the field's never matches in the
    reference: the adaptor passes an empty set for it. field_type "keyword": column is a keyword column
    (HostShard.keyword_columns) and values are its terms (str or bytes), matched as String.equals does (the TEXTTERMS set of
    an atom field); each searcher turns them into codes of its dictionary."""
    column: int
    values: tuple
    field_type: str = "long"

    def sortable(self) -> np.ndarray:
        """the values in the column's sortable-long domain"""
        if self.field_type == "float":
            return np.array([float_to_sortable_int(v) for v in self.values], np.int64)
        if self.field_type == "double":
            return np.array([double_to_sortable_long(v) for v in self.values], np.int64)
        return np.array([int(v) for v in self.values], np.int64)


@dataclass(frozen=True)
class FilterCollector:
    """FilterCollector (FilterCollectorManager): of the docs a query collects, those that pass `filter` are counted (the
    docCount) and handed to the nested collectors. filter: a flat query (BooleanQuery / TermQuery / RangeQuery /
    MatchAllDocsQuery; only matching counts) or a ValueSetFilter. nested: (name, TermsCollector | MinCollector | MaxCollector |
    SumCollector | TopHitsCollector | FilterCollector) pairs, at least one. Its result is {"doc_count": int32 [nq], name:
    the nested collector's result}: a terms or filter collector's own result, float64 [nq] (min / max / sum), or {"docs",
    "scores" [nq, top_hits - start_hit], "counts", "total_hits" [nq][, "sort_values" [nq, top_hits - start_hit, n_fields]]}
    (top hits)."""
    filter: object
    nested: tuple = ()


_VALUE_TYPE = {"int": 0, "long": 0, "float": 1, "double": 2, "keyword": 3}

# nrtgpu_index_keyword_range flags
_KW_NO_LOWER, _KW_NO_UPPER, _KW_LOWER_EXCLUSIVE, _KW_UPPER_EXCLUSIVE, _KW_PREFIX = 1, 2, 4, 8, 16


@dataclass(frozen=True)
class _KeywordCodeSet:
    """a keyword ValueSetFilter resolved by a searcher: the codes of its terms in the searcher's dictionary
    (NRTGPU_AGG_FILTER_KEYWORD_SET)"""
    column: int
    codes: tuple


def _keyword_range(fn, handle, column: int, q) -> Tuple[int, int]:
    """the code range of a KeywordRangeQuery / KeywordPrefixQuery through nrtgpu_index_keyword_range /
    nrtgpu_searcher_keyword_range (fn) on handle"""
    if isinstance(q, KeywordPrefixQuery):
        lower, upper, flags = _utf8_bytes(q.prefix), b"", _KW_PREFIX
    else:
        flags = 0
        lower = b"" if q.lower is None else _utf8_bytes(q.lower)
        upper = b"" if q.upper is None else _utf8_bytes(q.upper)
        flags |= _KW_NO_LOWER if q.lower is None else (0 if q.include_lower else _KW_LOWER_EXCLUSIVE)
        flags |= _KW_NO_UPPER if q.upper is None else (0 if q.include_upper else _KW_UPPER_EXCLUSIVE)
    lo, hi = C.c_int64(), C.c_int64()
    check(fn(handle, column, lower, len(lower), upper, len(upper), flags, C.byref(lo), C.byref(hi)))
    return lo.value, hi.value


def _resolve_keywords(q, searcher):
    """q with every KeywordRangeQuery / KeywordPrefixQuery turned into _KeywordCodes and every keyword ValueSetFilter into
    a _KeywordCodeSet by searcher.keyword_range / keyword_seek (its own dictionary), through BooleanQuery,
    DisjunctionMaxQuery, ConstantScoreQuery, MinScoreQuery, BoostQuery and FilterCollector; q itself when it holds none"""
    if isinstance(q, (KeywordRangeQuery, KeywordPrefixQuery)):
        return _KeywordCodes(q.column, *searcher.keyword_range(q))
    if isinstance(q, BoostQuery):
        sub = _resolve_keywords(q.query, searcher)
        return q if sub is q.query else BoostQuery(sub, q.boost)
    if isinstance(q, BooleanQuery):
        subs = [_resolve_keywords(c.query, searcher) for c in q.clauses]
        if all(x is c.query for x, c in zip(subs, q.clauses)):
            return q
        return BooleanQuery([BooleanClause(x, c.occur) for x, c in zip(subs, q.clauses)], q.minimum_number_should_match)
    if isinstance(q, DisjunctionMaxQuery):
        subs = [_resolve_keywords(d, searcher) for d in q.disjuncts]
        return q if all(x is d for x, d in zip(subs, q.disjuncts)) else DisjunctionMaxQuery(subs, q.tie_breaker)
    if isinstance(q, ConstantScoreQuery):
        sub = _resolve_keywords(q.filter, searcher)
        return q if sub is q.filter else ConstantScoreQuery(sub)
    if isinstance(q, MinScoreQuery):
        sub = _resolve_keywords(q.query, searcher)
        return q if sub is q.query else MinScoreQuery(sub, q.min_score)
    if isinstance(q, NestedQuery):
        sub = _resolve_keywords(q.query, searcher)
        return q if sub is q.query else NestedQuery(sub, q.path_term, q.score_mode)
    if isinstance(q, ValueSetFilter) and q.field_type == "keyword":
        return _KeywordCodeSet(q.column, tuple(searcher.keyword_seek(q.column, _utf8_bytes(v)) for v in q.values))
    if isinstance(q, FilterCollector):
        f = _resolve_keywords(q.filter, searcher)
        nested = tuple((name, _resolve_keywords(c, searcher)) for name, c in q.nested)
        if f is q.filter and all(x is c for (_, x), (_, c) in zip(nested, q.nested)):
            return q
        return FilterCollector(f, nested)
    return q


def _resolve_all(items, searcher):
    """_resolve_keywords over a sequence (None entries kept)"""
    return None if items is None else [None if x is None else _resolve_keywords(x, searcher) for x in items]


def _keyword_keys(collectors: Sequence[object], outs: Sequence[object], term, term_names=None) -> None:
    """Turns the ordinal keys of keyword terms collectors (and those nested in filter collectors) into str, and the
    "sort_values" of top hits sorted by a Sort with a keyword field into object arrays (_keyword_sort_values), in place;
    term(column, ord) -> bytes, term_names: the owner's _TermNames"""
    for c, o in zip(collectors, outs):
        if isinstance(c, TopHitsCollector):
            if c.sort is not None and "sort_values" in o:
                o["sort_values"] = _keyword_sort_values(c.sort_fields(), o["sort_values"], term_names)
            continue
        if isinstance(c, TermsCollector) and "nested" in o:
            tops = [(name, x) for name, x in c.nested if isinstance(x, TopHitsCollector)]
            _keyword_keys([x for _, x in tops], [o["nested"][name] for name, _ in tops], term, term_names)
        if isinstance(c, TermsCollector) and c.field_type == "keyword":
            filled = np.arange(o["keys"].shape[1])[None, :] < np.asarray(o["n"])[:, None]
            ords, at = np.unique(o["keys"][filled], return_inverse=True)   # one lookup per distinct term of the batch
            names = np.empty(len(ords), object)
            names[:] = [term(c.column, int(x)).decode("utf-8") for x in ords]
            keys = np.full(o["keys"].shape, None, object)
            keys[filled] = names[at.reshape(-1)]
            o["keys"] = keys
        elif isinstance(c, FilterCollector):
            nested_names = [name for name, x in c.nested]
            _keyword_keys([x for _, x in c.nested], [o[name] for name in nested_names], term, term_names)


def _term_bytes(fn, *args) -> bytes:
    """the bytes of one keyword term through nrtgpu_index_keyword_term / nrtgpu_searcher_keyword_term (fn bound to its
    handle, column and ordinal)"""
    n = C.c_int32()
    check(fn(*args, None, 0, C.byref(n)))
    buf = (C.c_uint8 * max(n.value, 1))()
    check(fn(*args, buf, n.value, C.byref(n)))
    return bytes(buf[:n.value])


@dataclass
class FieldDoc:
    doc: int
    value: object = 0   # fields[0], sortable-long domain; a keyword field's str, or None for no value
    values: Optional[Tuple[object, ...]] = None   # every field of a multi-field Sort (a row of SortedResult.sort_values)


@dataclass
class SortedResult:
    docs: np.ndarray          # int32 [nq, k]
    sort_values: np.ndarray   # int64 [nq, k] FieldDoc.fields[0] of every hit; [nq, k, n_fields] for a sequence of SortTypes;
                              # object (str / None for keyword fields, int else) when the Sort has a keyword field
    counts: np.ndarray
    total_hits: np.ndarray
    relation: np.ndarray
    hit_timeout: Optional[np.ndarray] = None        # uint8 [nq] (multi-field path)
    terminated_early: Optional[np.ndarray] = None   # uint8 [nq] (multi-field path)


def _f32(x: float) -> np.float32:
    return np.float32(x)


def _flatten(q, boost: np.float32, out: list, occur: Occur) -> None:
    """One clause of the flat BooleanQuery; BoostQuery boosts multiply outermost-first in float
    (BoostQuery.createWeight passes boost * this.boost down)."""
    q, boost = _unboost(q, boost)
    if isinstance(q, TermQuery):
        out.append((int(occur), 0, int(q.term), float(boost), 0, 0))
    elif isinstance(q, RangeQuery):
        out.append((int(occur), 1, int(q.column), float(boost), int(q.lower), int(q.upper)))
    elif isinstance(q, MatchAllDocsQuery):
        out.append((int(occur), 2, 0, float(boost), 0, 0))
    elif isinstance(q, _KeywordCodes):
        out.append((int(occur), 5, int(q.column), float(boost), int(q.lo), int(q.hi)))
    elif isinstance(q, (KeywordRangeQuery, KeywordPrefixQuery)):
        raise ValueError(f"{type(q).__name__} is resolved to codes by a searcher (GpuIndexSearcher / GpuLeafSearcher)")
    else:
        raise NrtGpuUnsupported(3, f"query node {type(q).__name__} is outside the GPU path")


def compile_queries(queries: Sequence[object], search_after: Optional[Sequence[Optional[ScoreDoc]]] = None):
    """Query trees -> (Clause[], Query[]) for nrtgpu_search_bool. A bare leaf is a single MUST clause
    (Lucene rewrites a one-clause BooleanQuery to its clause; scores are identical)."""
    flat, qs = [], []
    for i, q in enumerate(queries):
        q, boost = _unboost(q, _f32(1.0))
        begin = len(flat)
        msm = 0
        if isinstance(q, BooleanQuery):
            msm = q.minimum_number_should_match
            for cl in q.clauses:
                if isinstance(cl.query, BooleanQuery):
                    raise NrtGpuUnsupported(3, "nested BooleanQuery is outside the GPU path")
                _flatten(cl.query, boost, flat, cl.occur)
        else:
            _flatten(q, boost, flat, Occur.MUST)
        after = search_after[i] if search_after is not None else None
        qs.append((begin, len(flat), msm, 1 if after is not None else 0,
                   after.doc if after is not None else 0, after.score if after is not None else 0.0))
    carr = (Clause * max(len(flat), 1))()
    for i, (occ, kind, id_, b, lo, hi) in enumerate(flat):
        carr[i] = Clause(occ, kind, id_, b, lo, hi)
    qarr = (CQuery * max(len(qs), 1))()
    for i, t in enumerate(qs):
        qarr[i] = CQuery(*t)
    return carr, len(flat), qarr, len(qs)


def _unboost(q, boost: np.float32):
    """(the query under any BoostQuerys, the boost folded outermost first in float). A boost < 0 is refused as the
    reference refuses it (QueryNodeMapper.java:127), a NaN or infinite one as Lucene's BoostQuery does."""
    while isinstance(q, BoostQuery):
        if q.boost < 0:
            raise ValueError("Boost must be a positive number")
        if not math.isfinite(q.boost):
            raise ValueError(f"Boost must be a finite number, got {q.boost}")
        boost = _f32(boost * _f32(q.boost))
        q = q.query
    return q, boost


def compile_tree(queries: Sequence[object], search_after: Optional[Sequence[Optional[ScoreDoc]]] = None,
                 phrase_table: bool = False):
    """Query trees -> (Clause[], n_clauses, Node[], n_nodes, Query[], nq) for nrtgpu_search_tree. The root of a query is a
    BooleanQuery (a bare leaf, DisjunctionMaxQuery, ConstantScoreQuery or MinScoreQuery becomes its single MUST clause);
    every BooleanQuery, DisjunctionMaxQuery, ConstantScoreQuery or MinScoreQuery below it is a node, numbered in pre-order
    over the batch, whose clauses are one range of the clause array. BoostQuery boosts are folded through the nodes into
    the leaves, outermost first in float, so node clauses carry boost 1 (BoostQuery.createWeight passes boost * this.boost
    down). A ConstantScoreQuery or MinScoreQuery node takes the boost folded down to it as its own and the fold starts again
    at 1 below it; MinScoreQuery(q, 0) is compiled as q, and a min_score < 0 raises ValueError. A NestedQuery is a node of
    kind 6 (its score mode in min_should_match) over one MUST node, its child query BooleanQuery{FILTER path term, MUST
    query}; the boost folds through it.
    phrase_table: return (Clause[], n_clauses, Node[], n_nodes, Phrase[], n_phrases, PhraseTerm[], n_phrase_terms, Query[],
    nq) for nrtgpu_search_tree_phrases instead: a PhraseQuery leaf is a clause of kind 4 whose id indexes the phrase table,
    a MultiPhraseQuery (or MatchPhrasePrefixQuery, rewritten) one of kind 6. Without it either is refused."""
    flat, nodes, qs = [], [], []
    phrases, pterms = [], []

    def leaf(sub, sb, occ):
        if isinstance(sub, MatchPhrasePrefixQuery):
            sub = sub.rewrite()
        if isinstance(sub, MultiPhraseQuery):
            if not phrase_table:
                raise NrtGpuUnsupported(3, "MultiPhraseQuery needs compile_tree(..., phrase_table=True)")
            begin = len(pterms)
            pterms.extend(sub.term_positions())
            phrases.append((begin, len(pterms), int(sub.slop), 0))
            flat.append((int(occ), 6, len(phrases) - 1, float(sb), 0, 0))
        elif isinstance(sub, PhraseQuery):
            if not phrase_table:
                raise NrtGpuUnsupported(3, "PhraseQuery needs compile_tree(..., phrase_table=True)")
            begin = len(pterms)
            pterms.extend(sub.term_positions())
            phrases.append((begin, len(pterms), int(sub.slop), 0))
            flat.append((int(occ), 4, len(phrases) - 1, float(sb), 0, 0))
        else:
            _flatten(sub, sb, flat, occ)

    def unwrap(q, b):
        """_unboost, through MinScoreQuerys of threshold 0 (QueryNodeMapper returns their query unwrapped)"""
        while True:
            q, b = _unboost(q, b)
            if not isinstance(q, MinScoreQuery):
                return q, b
            if q.min_score < 0:
                raise ValueError("MinScoreQuery.min_score must be a non-negative number")
            if q.min_score != 0:
                return q, b
            q = q.query

    one = _f32(1.0)

    def parts(q, b):
        """(kind, clauses, msm, tie, the boost its clauses fold from, node boost, min_score) of a node reached with boost b"""
        if isinstance(q, BooleanQuery):
            return 0, [(c.query, c.occur) for c in q.clauses], q.minimum_number_should_match, 0.0, b, 0.0, 0.0
        if isinstance(q, DisjunctionMaxQuery):
            return 1, [(d, Occur.SHOULD) for d in q.disjuncts], 0, float(q.tie_breaker), b, 0.0, 0.0
        if isinstance(q, ConstantScoreQuery):
            return 3, [(q.filter, Occur.MUST)], 0, 0.0, one, float(b), 0.0
        if isinstance(q, NestedQuery):   # ToParentBlockJoinQuery.createWeight passes its boost to the child weight
            return 6, [(q.child_query(), Occur.MUST)], q.mode(), 0.0, b, 0.0, 0.0
        return 4, [(q.query, Occur.MUST)], 0, 0.0, one, float(b), float(q.min_score)

    for i, q in enumerate(queries):
        q, boost = unwrap(q, one)
        if isinstance(q, BooleanQuery):
            root = (0, [(c.query, c.occur) for c in q.clauses], q.minimum_number_should_match, 0.0, boost, 0.0, 0.0)
        else:
            root = (0, [(q, Occur.MUST)], 0, 0.0, boost, 0.0, 0.0)
        order = []   # pre-order: [kind, [(leaf, boost, occur) | (node position, None, occur)], msm, tie, node boost, min_score]

        def visit(kind, cls, msm, tie, b, nb, ms):
            pos = len(order)
            order.append(None)
            children = []
            for sub, occ in cls:
                s, sb = unwrap(sub, b)
                if isinstance(s, (BooleanQuery, DisjunctionMaxQuery, ConstantScoreQuery, MinScoreQuery, NestedQuery)):
                    children.append((visit(*parts(s, sb)), None, occ))
                else:
                    children.append((s, sb, occ))
            order[pos] = (kind, children, msm, tie, nb, ms)
            return pos

        visit(*root)
        base = len(nodes) - 1   # node id of pre-order position p > 0: base + p
        begin_end = []
        for kind, children, msm, tie, nb, ms in order:
            begin = len(flat)
            for sub, sb, occ in children:
                if sb is None:
                    flat.append((int(occ), 3, base + sub, 1.0, 0, 0))
                else:
                    leaf(sub, sb, occ)
            begin_end.append((begin, len(flat)))
        for p in range(1, len(order)):
            kind, _, msm, tie, nb, ms = order[p]
            nodes.append((kind, begin_end[p][0], begin_end[p][1], msm, tie, nb, ms))
        after = search_after[i] if search_after is not None else None
        qs.append((begin_end[0][0], begin_end[0][1], root[2], 1 if after is not None else 0,
                   after.doc if after is not None else 0, after.score if after is not None else 0.0))
    carr = (Clause * max(len(flat), 1))(*[Clause(*c) for c in flat])
    narr = (_native.Node * max(len(nodes), 1))(*[_native.Node(*n) for n in nodes])
    qarr = (CQuery * max(len(qs), 1))(*[CQuery(*t) for t in qs])
    if phrase_table:
        parr = (_native.Phrase * max(len(phrases), 1))(*[_native.Phrase(*p) for p in phrases])
        tarr = (_native.PhraseTerm * max(len(pterms), 1))(*[_native.PhraseTerm(*t) for t in pterms])
        return carr, len(flat), narr, len(nodes), parr, len(phrases), tarr, len(pterms), qarr, len(qs)
    return carr, len(flat), narr, len(nodes), qarr, len(qs)


def compile_filters(filter_queries: Sequence[Optional[object]], nq: int):
    """Per-query kNN filter queries (KnnQuery.filter; None = no filter) -> (Clause[], n_clauses, Query[], n_filters,
    filter_of int32[nq]) for nrtgpu_search_knn_filtered. Filters that compile to the same flat BooleanQuery, boosts aside
    (a filter only matches), share one index, so the device evaluates each of them once per call."""
    if len(filter_queries) != nq:
        raise ValueError(f"filter_queries has {len(filter_queries)} entries for {nq} query vectors")
    present = [i for i, f in enumerate(filter_queries) if f is not None]
    filter_of = np.full(nq, -1, np.int32)
    flat, qs, index_of = [], [], {}
    if present:
        carr, _, qarr, _ = compile_queries([filter_queries[i] for i in present])
        for j, i in enumerate(present):
            q = qarr[j]
            cls = tuple((c.occur, c.kind, c.id, c.boost, c.lo, c.hi) for c in carr[q.clause_begin:q.clause_end])
            key = (tuple(c[:3] + c[4:] for c in cls), q.min_should_match)
            if key not in index_of:
                index_of[key] = len(qs)
                qs.append((len(flat), len(flat) + len(cls), q.min_should_match, 0, 0, 0.0))
                flat.extend(cls)
            filter_of[i] = index_of[key]
    carr = (Clause * max(len(flat), 1))(*[Clause(*c) for c in flat])
    qarr = (CQuery * max(len(qs), 1))(*[CQuery(*t) for t in qs])
    return carr, len(flat), qarr, len(qs), filter_of


class GpuContext:
    def __init__(self, device: int = 0):
        self._lib = _native.gpu_lib()
        h = C.c_void_p()
        check(self._lib.nrtgpu_init(device, C.byref(h)))
        self.handle = h
        self.device = device

    def close(self):
        if self.handle:
            self._lib.nrtgpu_shutdown(self.handle)
            self.handle = None


class GpuIndex:
    """Device image of one shard at one reader version (ShardSearcherFactory.newSearcher hook)."""

    def __init__(self, ctx: GpuContext, shard: HostShard):
        self._lib = _native.gpu_lib()
        self.ctx = ctx
        pinned = PinnedDesc(shard)
        h = C.c_void_p()
        check(self._lib.nrtgpu_index_build(ctx.handle, C.byref(pinned.desc), C.byref(h)))
        self.handle = h
        self.n_docs, self.doc_base = shard.n_docs, shard.doc_base
        self._orders = {}
        self._terms = {}
        self.keyword_names = _TermNames(self.keyword_term)   # str of terms by ordinal (sorted pages' keyword values)
        if shard.post_positions is not None:
            self.add_positions(shard.post_positions)
        if shard.parent_term is not None:
            self.add_parents(shard.parent_term)
        if pinned.n_keyword:
            try:
                check(self._lib.nrtgpu_index_add_keyword_columns(self.handle, pinned.keyword, pinned.n_keyword))
            except Exception:   # a refused column: the image built above is freed, not leaked
                self.close()
                raise

    def keyword_term(self, column: int, ord_: int) -> bytes:
        """term `ord_` of keyword column `column` of this image (nrtgpu_index_keyword_term)"""
        key = (column, ord_)
        if key not in self._terms:
            self._terms[key] = _term_bytes(self._lib.nrtgpu_index_keyword_term, self.handle, column, ord_)
        return self._terms[key]

    def keyword_seek(self, column: int, term: bytes) -> int:
        """the sort code of `term` in keyword column `column` of this image (nrtgpu_index_keyword_seek): 2i + 2 for its
        term i, 2i + 1 for a term it does not hold"""
        return _seek(self._lib.nrtgpu_index_keyword_seek, self.handle, column, term)

    def keyword_range(self, q) -> Tuple[int, int]:
        """the code range [lo, hi] of a KeywordRangeQuery / KeywordPrefixQuery in this image's dictionary
        (nrtgpu_index_keyword_range)"""
        return _keyword_range(self._lib.nrtgpu_index_keyword_range, self.handle, q.column, q)

    def add_positions(self, positions: np.ndarray):
        """Term positions of every posting, posting after posting (HostShard.post_positions): what PhraseQuery needs."""
        p = np.ascontiguousarray(positions, np.int32)
        check(self._lib.nrtgpu_index_add_positions(self.handle, p.ctypes.data if len(p) else None, len(p)))

    def add_parents(self, root_term: int):
        """The parent docs of the image's blocks: the docs of `root_term` (HostShard.parent_term), what NestedQuery needs."""
        check(self._lib.nrtgpu_index_add_parents(self.handle, int(root_term)))

    def sort_order(self, fields: Sequence[SortType], stream: int = 0) -> C.c_void_p:
        """The nrtgpu_sort_order of a Sort, built on first use and kept until close(): it depends on the columns only, so
        deletes and statistics refreshes leave it valid."""
        cf = [f.c_field() for f in fields]
        key = tuple((f.kind, f.column, f.reverse, f.selector, f.missing_value) for f in cf)
        if key not in self._orders:
            arr = (_native.SortField * max(len(cf), 1))(*cf)
            h = C.c_void_p()
            check(self._lib.nrtgpu_sort_order_create(self.handle, arr, len(cf), C.c_void_p(stream), C.byref(h)))
            self._orders[key] = h
        return self._orders[key]

    def set_live_docs(self, live_docs: Optional[np.ndarray]):
        """Deletes of a new reader version (LeafReader.getLiveDocs): refreshed in place, no image rebuild."""
        lv = None if live_docs is None else np.ascontiguousarray(live_docs, np.uint8)
        check(self._lib.nrtgpu_index_set_live_docs(self.handle, None if lv is None else lv.ctypes.data))

    def update_stats(self, term_df: Optional[np.ndarray], field_doc_count: Sequence[int], field_sum_ttf: Sequence[int]):
        """Index-wide BM25 statistics changed (a leaf was added elsewhere in the shard): idf inputs, length caches, impacts."""
        df = None if term_df is None else np.ascontiguousarray(term_df, np.int64)
        dc = np.ascontiguousarray(field_doc_count, np.int64)
        tt = np.ascontiguousarray(field_sum_ttf, np.int64)
        check(self._lib.nrtgpu_index_update_stats(self.handle, None if df is None else df.ctypes.data, dc.ctypes.data, tt.ctypes.data))

    @property
    def device_bytes(self) -> int:
        return int(self._lib.nrtgpu_index_device_bytes(self.handle))

    def close(self):
        if self.handle:
            for h in self._orders.values():
                self._lib.nrtgpu_sort_order_close(h)
            self._orders.clear()
            self._lib.nrtgpu_index_close(self.handle)
            self.handle = None


@dataclass
class BatchResult:
    docs: np.ndarray      # int32 [nq, k]
    scores: np.ndarray    # float32 [nq, k]
    counts: np.ndarray    # int32 [nq]
    total_hits: np.ndarray  # int64 [nq]
    relation: np.ndarray  # uint8 [nq]
    hit_timeout: Optional[np.ndarray] = None        # uint8 [nq] (SearchResponse.hitTimeout, per query of the batch)
    terminated_early: Optional[np.ndarray] = None   # uint8 [nq] (SearchResponse.terminatedEarly)

    def top_docs(self, i: int) -> TopDocs:
        n = int(self.counts[i])
        return TopDocs(TotalHits(int(self.total_hits[i]), Relation(int(self.relation[i]))),
                       [ScoreDoc(int(d), float(s)) for d, s in zip(self.docs[i, :n], self.scores[i, :n])])


class PreparedBatch:
    """nrtgpu_batch: compiled batch resident on the device (launch many times, inputs stay in HBM)."""

    def __init__(self, index: GpuIndex, carr, ncl, qarr, nq, top_k, threshold, flags=0, nodes=None, phrases=None):
        """nodes: (Node[], n_nodes) of a query-tree batch (nrtgpu_batch_prepare_tree), None for flat queries; phrases:
        (Phrase[], n_phrases, PhraseTerm[], n_phrase_terms) of a tree batch with phrases (nrtgpu_batch_prepare_tree_phrases)."""
        self._lib = _native.gpu_lib()
        self.index, self.nq, self.top_k = index, nq, top_k
        h = C.c_void_p()
        if phrases is not None:
            check(self._lib.nrtgpu_batch_prepare_tree_phrases(index.handle, carr, ncl, nodes[0], nodes[1], *phrases, qarr, nq, top_k,
                                                              threshold, flags, C.byref(h)))
        elif nodes is None:
            check(self._lib.nrtgpu_batch_prepare(index.handle, carr, ncl, qarr, nq, top_k, threshold, flags, C.byref(h)))
        else:
            check(self._lib.nrtgpu_batch_prepare_tree(index.handle, carr, ncl, nodes[0], nodes[1], qarr, nq, top_k, threshold, flags,
                                                      C.byref(h)))
        self.handle = h

    def run(self, stream: int = 0):
        check(self._lib.nrtgpu_batch_run(self.handle, C.c_void_p(stream)))

    def fetch(self, stream: int = 0, out: Optional[BatchResult] = None) -> BatchResult:
        if out is None:
            out = BatchResult(np.zeros((self.nq, self.top_k), np.int32), np.zeros((self.nq, self.top_k), np.float32),
                              np.zeros(self.nq, np.int32), np.zeros(self.nq, np.int64), np.zeros(self.nq, np.uint8))
        check(self._lib.nrtgpu_batch_fetch(self.handle, C.c_void_p(stream), out.docs.ctypes.data, out.scores.ctypes.data,
                                           out.counts.ctypes.data, out.total_hits.ctypes.data, out.relation.ctypes.data))
        return out

    def stats(self):
        a, l, w = C.c_int64(), C.c_int32(), C.c_int64()
        check(self._lib.nrtgpu_batch_stats(self.handle, C.byref(a), C.byref(l), C.byref(w)))
        return {"alg_postings": a.value, "launches_per_run": l.value, "work_items": w.value}

    def stage_ms(self, stage: int) -> float:
        ms = C.c_float()
        check(self._lib.nrtgpu_batch_stage_ms(self.handle, stage, C.byref(ms)))
        return ms.value

    def reset_timing(self):
        check(self._lib.nrtgpu_batch_reset_timing(self.handle))

    def bind_output(self, d_docs: int, d_scores: int, d_counts: int):
        check(self._lib.nrtgpu_batch_bind_output(self.handle, C.c_void_p(d_docs), C.c_void_p(d_scores), C.c_void_p(d_counts)))

    def bind_packed(self, d_record: int):
        """Results of subsequent runs go into one packed DEVICE record (nrtgpu_batch_bind_packed): the buffer a multi-GPU
        step all-gathers."""
        check(self._lib.nrtgpu_batch_bind_packed(self.handle, C.c_void_p(d_record)))

    def device_results(self):
        d, s, c = C.c_void_p(), C.c_void_p(), C.c_void_p()
        check(self._lib.nrtgpu_batch_device_results(self.handle, C.byref(d), C.byref(s), C.byref(c)))
        return d.value, s.value, c.value

    def close(self):
        if self.handle:
            self._lib.nrtgpu_batch_free(self.handle)
            self.handle = None


def _collector_records(nq: int, additional: Sequence[object]):
    """The records of a batch's additional collectors (search_with_collectors of either searcher): the nrtgpu_aggregation and
    _result arrays, the nrtgpu_nested_aggregation and _result arrays of their terms collectors' nested collectors (None
    without any) and their count, and the result objects the call fills, one per collector."""
    aggs = (CAgg * len(additional))()
    res = (CAggResult * len(additional))()
    outs, nested, nested_res = [], [], []
    for i, a in enumerate(additional):
        vt = _VALUE_TYPE[a.field_type]
        if isinstance(a, TermsCollector):
            aggs[i] = CAgg(1, a.column, vt, a.size, 1 if a.order_desc else 0, 0)
            o = {"keys": np.zeros((nq, a.size), np.int64), "counts": np.zeros((nq, a.size), np.int32), "n": np.zeros(nq, np.int32),
                 "total_buckets": np.zeros(nq, np.int32), "other_counts": np.zeros(nq, np.int64)}
            res[i] = CAggResult(None, o["keys"].ctypes.data, o["counts"].ctypes.data, o["n"].ctypes.data,
                                o["total_buckets"].ctypes.data, o["other_counts"].ctypes.data)
            if a.nested or a.order_by is not None:
                o["nested"] = _nested_specs(i, a, nq, nested, nested_res)
        else:
            kind = 2 if isinstance(a, MinCollector) else 3 if isinstance(a, MaxCollector) else 4
            aggs[i] = CAgg(kind, a.column, vt, 0, 0, 0)
            o = np.zeros(nq, np.float64)
            res[i] = CAggResult(o.ctypes.data, None, None, None, None, None)
        outs.append(o)
    narr = (CNested * len(nested))(*nested) if nested else None
    nres = (CNestedResult * len(nested))(*nested_res) if nested else None
    return aggs, res, narr, nres, len(nested), outs


class _FilteredRecords:
    """The records of a batch whose additional collectors hold filter collectors or top hits that need more than a terms
    bucket by score (nrtgpu_search_bool_aggs_sorted_hits): every terms, min / max / sum and filter collector becomes an
    nrtgpu_aggregation, a terms or filter collector under a filter names it by filter_agg (parents before children), a min /
    max / sum / top hits under a filter is a nested collector of it, and each filter gets its nrtgpu_agg_filter record
    (filter queries compiled by compile_queries). A top-level TopHitsCollector is the nested top hits of an implicit
    FilterCollector(MatchAllDocsQuery()): one filter row and 4 B of codes per doc on the device. A sorted top hits gets its
    nrtgpu_nested_sort, the orders of its Sort from orders_of(fields) (one per image). outs: the result objects the call
    fills, one per top-level collector; args: the records in the order of nrtgpu_search_bool_aggs_filtered, sorted_args in
    that of nrtgpu_search_bool_aggs_sorted_hits."""

    def __init__(self, nq: int, additional: Sequence[object], orders_of=None):
        self.nq, self.orders_of = nq, orders_of
        self.aggs, self.res, self.filters, self.nested, self.nested_res, self.sorts = [], [], [], [], [], []
        self.filter_queries, self.keep = [], []
        self.outs = [self._add(a, 0) for a in additional]
        n = len(self.aggs)
        aggs, res = (CAgg * n)(*self.aggs), (CAggResult * n)(*self.res)
        filt = (CAggFilter * n)(*self.filters)
        narr = (CNested * len(self.nested))(*self.nested) if self.nested else None
        nres = (CNestedResult * len(self.nested))(*self.nested_res) if self.nested else None
        nsort = (CNestedSort * len(self.nested))(*self.sorts) if any(x.orders for x in self.sorts) else None
        fcarr, fncl, fqarr, fnq = compile_queries(self.filter_queries) if self.filter_queries else (None, 0, None, 0)
        self.args = (aggs, n, res, narr, len(self.nested), nres, filt, fcarr, fncl, fqarr, fnq)
        self.sorted_args = self.args[:6] + (nsort,) + self.args[6:]

    def _top_hits(self, c: "TopHitsCollector", parent: int, shape: tuple, orders_parent: int = 0) -> dict:
        return _top_hits_spec(c, parent, shape, self.nested, self.nested_res, orders_parent, self.sorts, self.orders_of, self.keep)

    def _add(self, a, filter_agg: int):
        nq, i = self.nq, len(self.aggs)
        self.filters.append(CAggFilter())
        if isinstance(a, TermsCollector):
            self.aggs.append(CAgg(1, a.column, _VALUE_TYPE[a.field_type], a.size, 1 if a.order_desc else 0, filter_agg))
            o = {"keys": np.zeros((nq, a.size), np.int64), "counts": np.zeros((nq, a.size), np.int32), "n": np.zeros(nq, np.int32),
                 "total_buckets": np.zeros(nq, np.int32), "other_counts": np.zeros(nq, np.int64)}
            self.res.append(CAggResult(None, o["keys"].ctypes.data, o["counts"].ctypes.data, o["n"].ctypes.data,
                                       o["total_buckets"].ctypes.data, o["other_counts"].ctypes.data))
            if a.nested or a.order_by is not None:
                o["nested"] = _nested_specs(i, a, nq, self.nested, self.nested_res, self.sorts, self.orders_of, self.keep)
            return o
        if isinstance(a, TopHitsCollector):   # top level: the nested top hits of FilterCollector(MatchAllDocsQuery())
            self.aggs.append(CAgg(6, 0, 0, 0, 0, 0))
            self.res.append(CAggResult(None, None, None, None, None, None))
            self.filters[i] = CAggFilter(1, len(self.filter_queries), 0, 0, None)
            self.filter_queries.append(MatchAllDocsQuery())
            return self._top_hits(a, i, (nq,))
        if isinstance(a, FilterCollector):
            self.aggs.append(CAgg(6, 0, 0, 0, 0, filter_agg))
            o = {"doc_count": np.zeros(nq, np.int32)}
            self.res.append(CAggResult(None, None, o["doc_count"].ctypes.data, None, None, None))
            f = a.filter
            if isinstance(f, (ValueSetFilter, _KeywordCodeSet)):
                keyword = isinstance(f, _KeywordCodeSet)
                if not keyword and f.field_type == "keyword":
                    raise ValueError("a keyword ValueSetFilter is resolved to codes by a searcher")
                vals = np.ascontiguousarray(np.array(f.codes, np.int64) if keyword else f.sortable(), np.int64)
                self.keep.append(vals)
                self.filters[i] = CAggFilter(4 if keyword else 2, 0, f.column, len(vals), vals.ctypes.data if len(vals) else None)
            else:
                self.filters[i] = CAggFilter(1, len(self.filter_queries), 0, 0, None)
                self.filter_queries.append(f)
            names = [name for name, _ in a.nested]
            if len(set(names)) != len(names) or "doc_count" in names:
                raise ValueError("nested collector names must be unique and not 'doc_count'")
            for name, c in a.nested:
                if isinstance(c, (TermsCollector, FilterCollector)):
                    o[name] = self._add(c, i + 1)
                elif isinstance(c, TopHitsCollector):
                    o[name] = self._top_hits(c, i, (nq,))
                elif isinstance(c, (MinCollector, MaxCollector, SumCollector)):
                    kind = 2 if isinstance(c, MinCollector) else 3 if isinstance(c, MaxCollector) else 4
                    r = np.zeros(nq, np.float64)
                    self.nested.append(CNested(i, kind, c.column, _VALUE_TYPE[c.field_type], 0, 0, 0, 0))
                    self.nested_res.append(CNestedResult(r.ctypes.data, None, None, None, None))
                    self.sorts.append(CNestedSort())
                    o[name] = r
                else:
                    raise ValueError(f"nested collector {name!r}: {type(c).__name__} is not on the GPU path")
            return o
        kind = 2 if isinstance(a, MinCollector) else 3 if isinstance(a, MaxCollector) else 4
        self.aggs.append(CAgg(kind, a.column, _VALUE_TYPE[a.field_type], 0, 0, 0))
        o = np.zeros(nq, np.float64)
        self.res.append(CAggResult(o.ctypes.data, None, None, None, None, None))
        return o


def _has_filter(additional: Sequence[object]) -> bool:
    """whether the request takes the filtered records (_FilteredRecords): a filter collector, a top-level top hits, or a
    top hits with a Sort anywhere"""
    def sorted_hits(c) -> bool:
        if isinstance(c, TopHitsCollector):
            return c.sort is not None
        return isinstance(c, (TermsCollector, FilterCollector)) and any(sorted_hits(x) for _, x in c.nested)
    return any(isinstance(a, (FilterCollector, TopHitsCollector)) or sorted_hits(a) for a in additional)


def _top_hits_spec(c: TopHitsCollector, parent: int, shape: tuple, nested: list, nested_res: list, orders_parent: int = 0,
                   sorts: Optional[list] = None, orders_of=None, keep: Optional[list] = None) -> dict:
    """the nrtgpu_nested_aggregation record and result buffers of top hits collector c under aggregation `parent` (appended
    to nested / nested_res; its nrtgpu_nested_sort to sorts, when the call takes them); shape: the result's leading
    dimensions ([nq, size] under a terms collector, [nq] else); returns the result dict they fill"""
    w = max(c.top_hits - c.start_hit, 0)
    r = {"docs": np.zeros(shape + (w,), np.int32), "scores": np.zeros(shape + (w,), np.float32),
         "counts": np.zeros(shape, np.int32), "total_hits": np.zeros(shape, np.int64)}
    nested.append(CNested(parent, 5, 0, 0, c.top_hits, c.start_hit, orders_parent, 0))
    nested_res.append(CNestedResult(None, r["docs"].ctypes.data, r["scores"].ctypes.data, r["counts"].ctypes.data,
                                    r["total_hits"].ctypes.data))
    ns = CNestedSort()
    if c.sort is not None:
        fields = c.sort_fields()
        orders = orders_of(fields)
        keep.append(orders)
        r["sort_values"] = np.zeros(shape + (w, len(fields)), np.int64)
        ns = CNestedSort(C.cast(orders, C.c_void_p), r["sort_values"].ctypes.data)
    if sorts is not None:
        sorts.append(ns)
    return r


def _nested_specs(parent: int, a: TermsCollector, nq: int, nested: list, nested_res: list, sorts: Optional[list] = None,
                  orders_of=None, keep: Optional[list] = None) -> dict:
    """the nrtgpu_nested_aggregation records and result buffers of terms collector `parent` (appended to nested /
    nested_res, and their nrtgpu_nested_sort to sorts when the call takes them); returns the result dict they fill"""
    names = [name for name, _ in a.nested]
    if len(set(names)) != len(names):
        raise ValueError("nested collector names must be unique")
    if a.order_by is not None and a.order_by not in names:
        raise ValueError(f"order_by {a.order_by!r} is not a nested collector")
    o = {}
    for name, c in a.nested:
        if isinstance(c, TopHitsCollector):
            r = _top_hits_spec(c, parent, (nq, a.size), nested, nested_res, 1 if name == a.order_by else 0, sorts, orders_of, keep)
        elif isinstance(c, (MinCollector, MaxCollector, SumCollector)):
            kind = 2 if isinstance(c, MinCollector) else 3 if isinstance(c, MaxCollector) else 4
            r = np.zeros((nq, a.size), np.float64)
            nested.append(CNested(parent, kind, c.column, _VALUE_TYPE[c.field_type], 0, 0, 1 if name == a.order_by else 0, 0))
            nested_res.append(CNestedResult(r.ctypes.data, None, None, None, None))
            if sorts is not None:
                sorts.append(CNestedSort())
        else:
            raise ValueError(f"nested collector {name!r}: {type(c).__name__} is not on the GPU path")
        o[name] = r
    return o


class GpuIndexSearcher:
    """Batched stand-in for MyIndexSearcher.search(Query, CollectorManager)."""

    def __init__(self, index: GpuIndex):
        self._lib = _native.gpu_lib()
        self.index = index

    def prepare(self, queries: Sequence[object], collector: RelevanceCollector,
                search_after: Optional[Sequence[Optional[ScoreDoc]]] = None, flags: int = 0) -> PreparedBatch:
        if search_after is None and collector.search_after is not None:
            search_after = [collector.search_after] * len(queries)
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self.index), search_after)
        return PreparedBatch(self.index, carr, ncl, qarr, nq, collector.num_hits_to_collect,
                             collector.total_hits_threshold, flags)

    def search_batch(self, queries: Sequence[object], collector: RelevanceCollector,
                     search_after: Optional[Sequence[Optional[ScoreDoc]]] = None, stream: int = 0) -> BatchResult:
        """One call through the C ABI with HOST buffers (nrtgpu_search_bool)."""
        if search_after is None and collector.search_after is not None:
            search_after = [collector.search_after] * len(queries)
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self.index), search_after)
        k = collector.num_hits_to_collect
        out = BatchResult(np.zeros((nq, max(k, 1)), np.int32), np.zeros((nq, max(k, 1)), np.float32),
                          np.zeros(nq, np.int32), np.zeros(nq, np.int64), np.zeros(nq, np.uint8),
                          np.zeros(nq, np.uint8), np.zeros(nq, np.uint8))
        lim = collector.limits()
        check(self._lib.nrtgpu_search_bool_ex(self.index.handle, carr, ncl, qarr, nq, k, collector.total_hits_threshold, 0,
                                              None if lim is None else C.byref(lim), C.c_void_p(stream), out.docs.ctypes.data,
                                              out.scores.ctypes.data, out.counts.ctypes.data, out.total_hits.ctypes.data,
                                              out.relation.ctypes.data, out.hit_timeout.ctypes.data,
                                              out.terminated_early.ctypes.data))
        return out

    def prepare_tree(self, queries: Sequence[object], collector: RelevanceCollector,
                     search_after: Optional[Sequence[Optional[ScoreDoc]]] = None, flags: int = 0) -> PreparedBatch:
        """prepare() for queries that may nest BooleanQuery and DisjunctionMaxQuery (nrtgpu_batch_prepare_tree)."""
        if search_after is None and collector.search_after is not None:
            search_after = [collector.search_after] * len(queries)
        carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(_resolve_all(queries, self.index), search_after, phrase_table=True)
        return PreparedBatch(self.index, carr, ncl, qarr, nq, collector.num_hits_to_collect, collector.total_hits_threshold, flags,
                             nodes=(narr, nn), phrases=(parr, n_ph, tarr, n_pt) if n_ph else None)

    def search_tree(self, queries: Sequence[object], collector: RelevanceCollector,
                    search_after: Optional[Sequence[Optional[ScoreDoc]]] = None, stream: int = 0) -> BatchResult:
        """search_batch() for queries that may nest BooleanQuery and DisjunctionMaxQuery (nrtgpu_search_tree): a batch with a
        nested query or a PhraseQuery runs on the window engine (phrases: nrtgpu_search_tree_phrases)."""
        if search_after is None and collector.search_after is not None:
            search_after = [collector.search_after] * len(queries)
        carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(_resolve_all(queries, self.index), search_after, phrase_table=True)
        k = collector.num_hits_to_collect
        out = BatchResult(np.zeros((nq, max(k, 1)), np.int32), np.zeros((nq, max(k, 1)), np.float32),
                          np.zeros(nq, np.int32), np.zeros(nq, np.int64), np.zeros(nq, np.uint8),
                          np.zeros(nq, np.uint8), np.zeros(nq, np.uint8))
        lim = collector.limits()
        outs = (None if lim is None else C.byref(lim), C.c_void_p(stream), out.docs.ctypes.data, out.scores.ctypes.data,
                out.counts.ctypes.data, out.total_hits.ctypes.data, out.relation.ctypes.data, out.hit_timeout.ctypes.data,
                out.terminated_early.ctypes.data)
        if n_ph:
            check(self._lib.nrtgpu_search_tree_phrases(self.index.handle, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, k,
                                                       collector.total_hits_threshold, 0, *outs))
        else:
            check(self._lib.nrtgpu_search_tree(self.index.handle, carr, ncl, narr, nn, qarr, nq, k, collector.total_hits_threshold, 0,
                                               *outs))
        return out

    def knn_query(self, queries: np.ndarray, knn: KnnQuery, sim: int, boosts: Optional[np.ndarray] = None,
                  filter_docs: Optional[np.ndarray] = None, stream: int = 0,
                  filter_queries: Optional[Sequence[Optional[object]]] = None):
        """KnnUtils.resolveKnnQueryAndBoost (:47-66) for a batch of query vectors under one KnnQuery configuration;
        filter_queries: the KnnQuery.filter of each query vector, or None (KnnUtils.java:135-155)."""
        knn.validate()
        docs, scores, counts = self.knn(queries, knn.k, boosts, filter_docs, stream, filter_queries)
        if knn.similarity_threshold is not None:   # MinThresholdQuery: drop hits scoring below the threshold's score
            th = similarity_to_score(knn.similarity_threshold, sim, queries.shape[1])
            for q in range(len(counts)):
                b = np.float32(1.0) if boosts is None else np.float32(boosts[q])
                keep = scores[q, :counts[q]] >= th * b
                n = int(keep.sum())
                docs[q, :n] = docs[q, :counts[q]][keep]; scores[q, :n] = scores[q, :counts[q]][keep]
                docs[q, n:] = 0; scores[q, n:] = 0; counts[q] = n
        return docs, scores, counts

    def search_sorted(self, queries: Sequence[object], collector: SortFieldCollector,
                      search_after: Optional[Sequence[Optional[FieldDoc]]] = None, stream: int = 0) -> SortedResult:
        """IndexSearcher.search(query, TopFieldCollectorManager(sort, numHits, after, threshold)) for a batch."""
        st = collector.sort
        if isinstance(st, SortType) and st.keyword:   # a one-field keyword Sort: a one-field order, sort_values [nq, k]
            out = self._search_sorted_fields(queries, collector, [st], search_after, stream)
            out.sort_values = out.sort_values.reshape(out.sort_values.shape[:2])
            return out
        if not isinstance(st, SortType) or st.field == "score":
            return self._search_sorted_fields(queries, collector, [st] if isinstance(st, SortType) else list(st), search_after, stream)
        after_sd = None if search_after is None else [None if a is None else ScoreDoc(a.doc, 0.0) for a in search_after]
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self.index), after_sd)
        k = collector.num_hits_to_collect
        out = SortedResult(np.zeros((nq, k), np.int32), np.zeros((nq, k), np.int64), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
                           np.zeros(nq, np.uint8))
        av = None
        if search_after is not None:
            av = np.array([0 if a is None else a.value for a in search_after], np.int64)
        docid = st.field == "docid"
        cs = CSort(2 if docid else 1, 0 if docid else int(st.field), 1 if st.reverse else 0, 0, 0 if docid else st.missing_value(),
                   None if av is None else av.ctypes.data)
        lim = None
        if collector.timeout_sec > 0 or collector.terminate_after > 0:
            lim = SearchLimits(collector.timeout_sec, 0.0, 0, collector.terminate_after, 0)
        check(self._lib.nrtgpu_search_sorted(self.index.handle, carr, ncl, qarr, nq, k, 0, C.byref(cs), None if lim is None else C.byref(lim),
                                             C.c_void_p(stream), out.docs.ctypes.data, out.sort_values.ctypes.data, out.counts.ctypes.data,
                                             out.total_hits.ctypes.data, out.relation.ctypes.data, None, None))
        return out

    def _search_sorted_fields(self, queries, collector: SortFieldCollector, fields: List[SortType],
                              search_after: Optional[Sequence[Optional[FieldDoc]]], stream: int) -> SortedResult:
        """A Sort of several fields (nrtgpu_search_sorted_fields) through the index's cached order of that Sort."""
        order = self.index.sort_order(fields, stream)
        nf = len(fields)
        after_sd = None if search_after is None else [None if a is None else ScoreDoc(a.doc, 0.0) for a in search_after]
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self.index), after_sd)
        k = collector.num_hits_to_collect
        out = SortedResult(np.zeros((nq, k), np.int32), np.zeros((nq, k, nf), np.int64), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
                           np.zeros(nq, np.uint8), np.zeros(nq, np.uint8), np.zeros(nq, np.uint8))
        av = None
        if search_after is not None:
            av = np.zeros((nq, nf), np.int64)
            for i, a in enumerate(search_after):
                if a is not None:
                    av[i] = _after_row(fields, a, self.index.keyword_seek)
        lim = None
        if collector.timeout_sec > 0 or collector.terminate_after > 0:
            lim = SearchLimits(collector.timeout_sec, 0.0, 0, collector.terminate_after, 0)
        check(self._lib.nrtgpu_search_sorted_fields(self.index.handle, order, carr, ncl, qarr, nq, k, 0,
                                                    None if av is None else av.ctypes.data, None if lim is None else C.byref(lim),
                                                    C.c_void_p(stream), out.docs.ctypes.data, out.sort_values.ctypes.data,
                                                    out.counts.ctypes.data, out.total_hits.ctypes.data, out.relation.ctypes.data,
                                                    out.hit_timeout.ctypes.data, out.terminated_early.ctypes.data))
        out.sort_values = _keyword_sort_values(fields, out.sort_values, self.index.keyword_names)
        return out

    def search_with_collectors(self, queries: Sequence[object], collector: RelevanceCollector, additional: Sequence[object],
                               stream: int = 0):
        """IndexSearcher.search with additional collectors (SearchCollectorManager fan-out): returns (BatchResult, results)
        where results[i] is a float64 [nq] array (min / max / sum) or a dict of bucket arrays (terms). A terms collector with
        nested collectors adds "nested": {name: float64 [nq, size] (min / max / sum) or {"docs", "scores" [nq, size,
        top_hits - start_hit], "counts", "total_hits" [nq, size][, "sort_values" [nq, size, top_hits - start_hit, n_fields]]}
        (top hits)}, per returned bucket. A FilterCollector's and a top-level TopHitsCollector's results are the dicts their
        docstrings describe (nrtgpu_search_bool_aggs_sorted_hits)."""
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self.index))
        k = collector.num_hits_to_collect
        out = BatchResult(np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
                          np.zeros(nq, np.uint8))
        hits = (out.docs.ctypes.data, out.scores.ctypes.data, out.counts.ctypes.data, out.total_hits.ctypes.data)
        if _has_filter(additional):   # filter collectors, top-level or sorted top hits: the records of _FilteredRecords
            fr = _FilteredRecords(nq, _resolve_all(additional, self.index), lambda fields: (C.c_void_p * 1)(self.index.sort_order(fields, stream).value))
            check(self._lib.nrtgpu_search_bool_aggs_sorted_hits(self.index.handle, carr, ncl, qarr, nq, k, 0, *fr.sorted_args,
                                                                C.c_void_p(stream), *hits))
            _keyword_keys(additional, fr.outs, self.index.keyword_term, self.index.keyword_names)
            return out, fr.outs
        aggs, res, narr, nres, n_nested, outs = _collector_records(nq, additional)
        if n_nested:
            check(self._lib.nrtgpu_search_bool_aggs_nested(self.index.handle, carr, ncl, qarr, nq, k, 0, aggs, len(additional), res,
                                                           narr, n_nested, nres, C.c_void_p(stream), *hits))
        else:
            check(self._lib.nrtgpu_search_bool_aggs(self.index.handle, carr, ncl, qarr, nq, k, 0, aggs, len(additional), res,
                                                    C.c_void_p(stream), *hits))
        _keyword_keys(additional, outs, self.index.keyword_term, self.index.keyword_names)
        return out, outs

    def search_tree_with_collectors(self, queries: Sequence[object], collector: RelevanceCollector, additional: Sequence[object],
                                    stream: int = 0):
        """search_with_collectors() for the queries of search_tree(): nested BooleanQuery and DisjunctionMaxQuery, PhraseQuery
        leaves, and flat batches of any width (nrtgpu_search_tree_aggs). The same collectors, the same (BatchResult, results)
        return; a batch with a nested query or a phrase, or a wide one, is collected by the window engine."""
        carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(_resolve_all(queries, self.index), phrase_table=True)
        k = collector.num_hits_to_collect
        out = BatchResult(np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
                          np.zeros(nq, np.uint8))
        fr = _FilteredRecords(nq, _resolve_all(additional, self.index), lambda fields: (C.c_void_p * 1)(self.index.sort_order(fields, stream).value))
        check(self._lib.nrtgpu_search_tree_aggs(self.index.handle, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, k, 0,
                                                *fr.sorted_args, C.c_void_p(stream), out.docs.ctypes.data, out.scores.ctypes.data,
                                                out.counts.ctypes.data, out.total_hits.ctypes.data))
        _keyword_keys(additional, fr.outs, self.index.keyword_term, self.index.keyword_names)
        return out, fr.outs

    def score_docs(self, queries: Sequence[object], docs: np.ndarray, counts: Optional[np.ndarray] = None, stream: int = 0):
        """Second pass of QueryRescorer: query q on its own hit list -> (matches uint8 [nq, n], scores float32 [nq, n])."""
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self.index))
        d = np.ascontiguousarray(docs, np.int32)
        cn = None if counts is None else np.ascontiguousarray(counts, np.int32)
        m, s = np.zeros(d.shape, np.uint8), np.zeros(d.shape, np.float32)
        check(self._lib.nrtgpu_score_docs(self.index.handle, carr, ncl, qarr, nq, d.shape[1], d.ctypes.data, None if cn is None else cn.ctypes.data,
                                          C.c_void_p(stream), m.ctypes.data, s.ctypes.data))
        return m, s

    def rescore_query(self, queries: Sequence[object], docs: np.ndarray, scores: np.ndarray, counts: np.ndarray, window: int,
                      query_weight: float, rescore_weight: float, stream: int = 0):
        """QueryRescore (QueryRescore.java:39-57) end to end on the device: returns docs, scores, counts of the rescored lists."""
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self.index))
        d = np.ascontiguousarray(docs, np.int32).copy()
        s = np.ascontiguousarray(scores, np.float32).copy()
        cn = np.ascontiguousarray(counts, np.int32)
        oc = np.zeros(nq, np.int32)
        check(self._lib.nrtgpu_rescore_query(self.index.handle, carr, ncl, qarr, nq, d.shape[1], cn.ctypes.data, window, query_weight,
                                             rescore_weight, C.c_void_p(stream), d.ctypes.data, s.ctypes.data, oc.ctypes.data))
        return d, s, oc

    def score_docs_tree(self, queries: Sequence[object], docs: np.ndarray, counts: Optional[np.ndarray] = None, stream: int = 0):
        """score_docs() for rescore queries that may nest BooleanQuery and DisjunctionMaxQuery or hold PhraseQuery leaves
        (nrtgpu_score_docs_tree): the queries search_tree takes."""
        carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(_resolve_all(queries, self.index), phrase_table=True)
        d = np.ascontiguousarray(docs, np.int32)
        cn = None if counts is None else np.ascontiguousarray(counts, np.int32)
        m, s = np.zeros(d.shape, np.uint8), np.zeros(d.shape, np.float32)
        check(self._lib.nrtgpu_score_docs_tree(self.index.handle, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, d.shape[1],
                                               d.ctypes.data, None if cn is None else cn.ctypes.data, C.c_void_p(stream),
                                               m.ctypes.data, s.ctypes.data))
        return m, s

    def rescore_query_tree(self, queries: Sequence[object], docs: np.ndarray, scores: np.ndarray, counts: np.ndarray, window: int,
                           query_weight: float, rescore_weight: float, stream: int = 0):
        """rescore_query() for rescore queries that may nest BooleanQuery and DisjunctionMaxQuery or hold PhraseQuery leaves
        (nrtgpu_rescore_query_tree): returns docs, scores, counts of the rescored lists."""
        carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(_resolve_all(queries, self.index), phrase_table=True)
        d = np.ascontiguousarray(docs, np.int32).copy()
        s = np.ascontiguousarray(scores, np.float32).copy()
        cn = np.ascontiguousarray(counts, np.int32)
        oc = np.zeros(nq, np.int32)
        check(self._lib.nrtgpu_rescore_query_tree(self.index.handle, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, d.shape[1],
                                                  cn.ctypes.data, window, query_weight, rescore_weight, C.c_void_p(stream),
                                                  d.ctypes.data, s.ctypes.data, oc.ctypes.data))
        return d, s, oc

    def fetch_columns(self, columns: Sequence[int], docs: np.ndarray, stream: int = 0):
        """Fetch phase on doc-value columns: values int64 [n_cols, n], has uint8 [n_cols, n] for the hits `docs`."""
        cols = np.ascontiguousarray(columns, np.int32)
        d = np.ascontiguousarray(docs, np.int32).reshape(-1)
        vals, has = np.zeros((len(cols), len(d)), np.int64), np.zeros((len(cols), len(d)), np.uint8)
        check(self._lib.nrtgpu_fetch_columns(self.index.handle, cols.ctypes.data, len(cols), d.ctypes.data, len(d), C.c_void_p(stream),
                                             vals.ctypes.data, has.ctypes.data))
        return vals, has

    def search(self, query, collector: RelevanceCollector) -> TopDocs:
        return self.search_batch([query], collector).top_docs(0)

    def knn(self, queries: np.ndarray, k: int, boosts: Optional[np.ndarray] = None,
            filter_docs: Optional[np.ndarray] = None, stream: int = 0, filter_queries: Optional[Sequence[Optional[object]]] = None):
        """Exact kNN (KnnUtils.resolveKnnQueryAndBoost with ExactVectorQuery semantics): returns docs, scores, counts.
        filter_docs: one 0/1 byte per doc, shared by the batch. filter_queries: one query object (KnnQuery.filter) or None per
        query vector, evaluated on the device."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        nq = q.shape[0]
        docs = np.zeros((nq, k), np.int32)
        scores = np.zeros((nq, k), np.float32)
        counts = np.zeros(nq, np.int32)
        b = None if boosts is None else np.ascontiguousarray(boosts, dtype=np.float32)
        # a kNN boost is a BoostQuery boost (KnnUtils.java:62-64); the rank-safety certificate needs score * boost monotone
        if b is not None and not (np.isfinite(b) & ~np.signbit(b)).all():
            raise ValueError("Boost must be a positive number")
        if filter_queries is not None:
            if filter_docs is not None:
                raise ValueError("pass filter_docs or filter_queries, not both")
            carr, ncl, qarr, nf, filter_of = compile_filters(_resolve_all(filter_queries, self.index), nq)
            check(self._lib.nrtgpu_search_knn_filtered(self.index.handle, q.ctypes.data, nq, k, None if b is None else b.ctypes.data,
                                                       carr, ncl, qarr, nf, filter_of.ctypes.data, C.c_void_p(stream),
                                                       docs.ctypes.data, scores.ctypes.data, counts.ctypes.data))
            return docs, scores, counts
        f = None if filter_docs is None else np.ascontiguousarray(filter_docs, dtype=np.uint8)
        check(self._lib.nrtgpu_search_knn(self.index.handle, q.ctypes.data, nq, k,
                                          None if b is None else b.ctypes.data, None if f is None else f.ctypes.data,
                                          C.c_void_p(stream), docs.ctypes.data, scores.ctypes.data, counts.ctypes.data))
        return docs, scores, counts


class GpuLeafSearcher:
    """IndexSearcher over the leaf images of one reader version (nrtgpu_searcher_*): every leaf runs the batch, pages are
    merged on the device (TopDocs.merge). A new NRT reader version = the old leaves' images + images of the new leaves."""

    def __init__(self, ctx: GpuContext, leaves: Sequence[GpuIndex]):
        self._lib = _native.gpu_lib()
        arr = (C.c_void_p * len(leaves))(*[l.handle for l in leaves])
        h = C.c_void_p()
        check(self._lib.nrtgpu_searcher_create(ctx.handle, arr, len(leaves), C.byref(h)))
        self.handle, self.leaves = h, list(leaves)
        self._terms = {}
        self.keyword_names = _TermNames(self.keyword_term)   # str of reader-wide terms by ordinal

    def keyword_term(self, column: int, ord_: int) -> bytes:
        """reader-wide term `ord_` of keyword column `column`: the byte-order union of the leaves' dictionaries
        (nrtgpu_searcher_keyword_term)"""
        key = (column, ord_)
        if key not in self._terms:
            self._terms[key] = _term_bytes(lambda *a: self._lib.nrtgpu_searcher_keyword_term(*a, None), self.handle, column, ord_)
        return self._terms[key]

    def keyword_seek(self, column: int, term: bytes) -> int:
        """the sort code of `term` in the reader-wide dictionary of keyword column `column` (nrtgpu_searcher_keyword_seek)"""
        return _seek(self._lib.nrtgpu_searcher_keyword_seek, self.handle, column, term)

    def keyword_range(self, q) -> Tuple[int, int]:
        """the code range [lo, hi] of a KeywordRangeQuery / KeywordPrefixQuery in the reader-wide dictionary
        (nrtgpu_searcher_keyword_range)"""
        return _keyword_range(self._lib.nrtgpu_searcher_keyword_range, self.handle, q.column, q)

    def search_batch(self, queries: Sequence[object], collector: RelevanceCollector, stream: int = 0,
                     search_after: Optional[Sequence[Optional[ScoreDoc]]] = None) -> BatchResult:
        """search_after: one reader-wide ScoreDoc (or None) per query; every leaf pages after it (TopDocs.merge of the pages)."""
        if search_after is None and collector.search_after is not None:
            search_after = [collector.search_after] * len(queries)
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self), search_after)
        k = collector.num_hits_to_collect
        out = BatchResult(np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
                          np.zeros(nq, np.uint8))
        lim = collector.limits()
        check(self._lib.nrtgpu_searcher_search_bool(self.handle, carr, ncl, qarr, nq, k, collector.total_hits_threshold, 0,
                                                    None if lim is None else C.byref(lim), C.c_void_p(stream), out.docs.ctypes.data,
                                                    out.scores.ctypes.data, out.counts.ctypes.data, out.total_hits.ctypes.data,
                                                    out.relation.ctypes.data))
        return out

    def search_sorted(self, queries: Sequence[object], collector: SortFieldCollector,
                      search_after: Optional[Sequence[Optional[FieldDoc]]] = None, stream: int = 0) -> SortedResult:
        """GpuIndexSearcher.search_sorted over the leaves (nrtgpu_searcher_search_sorted_fields): every leaf searches with its
        cached order of the Sort (GpuIndex.sort_order), the pages are merged on the device (TopFieldDocs.merge). A one-field
        Sort runs as a one-field order and returns sort_values [nq, k], as the single-image search does; search_after holds
        reader-wide FieldDocs."""
        st = collector.sort
        fields = [st] if isinstance(st, SortType) else list(st)
        orders = (C.c_void_p * len(self.leaves))(*[l.sort_order(fields, stream).value for l in self.leaves])
        nf = len(fields)
        after_sd = None if search_after is None else [None if a is None else ScoreDoc(a.doc, 0.0) for a in search_after]
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self), after_sd)
        k = collector.num_hits_to_collect
        out = SortedResult(np.zeros((nq, k), np.int32), np.zeros((nq, k, nf), np.int64), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
                           np.zeros(nq, np.uint8), np.zeros(nq, np.uint8), np.zeros(nq, np.uint8))
        av = None
        if search_after is not None:
            av = np.zeros((nq, nf), np.int64)
            for i, a in enumerate(search_after):
                if a is not None:
                    av[i] = _after_row(fields, a, self.keyword_seek)
        lim = None
        if collector.timeout_sec > 0 or collector.terminate_after > 0:
            lim = SearchLimits(collector.timeout_sec, 0.0, 0, collector.terminate_after, 0)
        check(self._lib.nrtgpu_searcher_search_sorted_fields(self.handle, orders, len(self.leaves), carr, ncl, qarr, nq, k, 0,
                                                             None if av is None else av.ctypes.data,
                                                             None if lim is None else C.byref(lim), C.c_void_p(stream),
                                                             out.docs.ctypes.data, out.sort_values.ctypes.data, out.counts.ctypes.data,
                                                             out.total_hits.ctypes.data, out.relation.ctypes.data,
                                                             out.hit_timeout.ctypes.data, out.terminated_early.ctypes.data))
        out.sort_values = _keyword_sort_values(fields, out.sort_values, self.keyword_names)
        if isinstance(st, SortType) and st.field != "score":
            out.sort_values = out.sort_values.reshape(nq, k)
        return out

    def search_tree(self, queries: Sequence[object], collector: RelevanceCollector,
                    search_after: Optional[Sequence[Optional[ScoreDoc]]] = None, stream: int = 0) -> BatchResult:
        """GpuIndexSearcher.search_tree over the leaves (nrtgpu_searcher_search_tree_phrases): query trees and phrases, the
        leaves' pages merged on the device (TopDocs.merge)."""
        if search_after is None and collector.search_after is not None:
            search_after = [collector.search_after] * len(queries)
        carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(_resolve_all(queries, self), search_after, phrase_table=True)
        k = collector.num_hits_to_collect
        out = BatchResult(np.zeros((nq, max(k, 1)), np.int32), np.zeros((nq, max(k, 1)), np.float32),
                          np.zeros(nq, np.int32), np.zeros(nq, np.int64), np.zeros(nq, np.uint8),
                          np.zeros(nq, np.uint8), np.zeros(nq, np.uint8))
        lim = collector.limits()
        check(self._lib.nrtgpu_searcher_search_tree_phrases(self.handle, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, k,
                                                            collector.total_hits_threshold, 0, None if lim is None else C.byref(lim),
                                                            C.c_void_p(stream), out.docs.ctypes.data, out.scores.ctypes.data,
                                                            out.counts.ctypes.data, out.total_hits.ctypes.data, out.relation.ctypes.data,
                                                            out.hit_timeout.ctypes.data, out.terminated_early.ctypes.data))
        return out

    def knn(self, queries: np.ndarray, k: int, boosts: Optional[np.ndarray] = None,
            filter_docs: Optional[np.ndarray] = None, stream: int = 0, filter_queries: Optional[Sequence[Optional[object]]] = None):
        """GpuIndexSearcher.knn over the leaves (nrtgpu_searcher_search_knn / _filtered): every leaf's exact top-k, merged by
        (score desc, doc asc) on the device. filter_docs: one 0/1 byte per global doc id of the reader."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        nq = q.shape[0]
        docs = np.zeros((nq, k), np.int32)
        scores = np.zeros((nq, k), np.float32)
        counts = np.zeros(nq, np.int32)
        b = None if boosts is None else np.ascontiguousarray(boosts, dtype=np.float32)
        if b is not None and not (np.isfinite(b) & ~np.signbit(b)).all():
            raise ValueError("Boost must be a positive number")
        if filter_queries is not None:
            if filter_docs is not None:
                raise ValueError("pass filter_docs or filter_queries, not both")
            carr, ncl, qarr, nf, filter_of = compile_filters(_resolve_all(filter_queries, self), nq)
            check(self._lib.nrtgpu_searcher_search_knn_filtered(self.handle, q.ctypes.data, nq, k, None if b is None else b.ctypes.data,
                                                                carr, ncl, qarr, nf, filter_of.ctypes.data, C.c_void_p(stream),
                                                                docs.ctypes.data, scores.ctypes.data, counts.ctypes.data))
            return docs, scores, counts
        f = None if filter_docs is None else np.ascontiguousarray(filter_docs, dtype=np.uint8)
        check(self._lib.nrtgpu_searcher_search_knn(self.handle, q.ctypes.data, nq, k, None if b is None else b.ctypes.data,
                                                   None if f is None else f.ctypes.data, C.c_void_p(stream),
                                                   docs.ctypes.data, scores.ctypes.data, counts.ctypes.data))
        return docs, scores, counts

    def search_with_collectors(self, queries: Sequence[object], collector: RelevanceCollector, additional: Sequence[object],
                               stream: int = 0):
        """GpuIndexSearcher.search_with_collectors over the leaves (nrtgpu_searcher_search_bool_aggs_nested): every leaf counts
        into reader-wide tables, buckets by value (the searcher's reader-wide dictionary of each terms column, built by the
        column's first aggregation), and the buckets, nested values and nested top hits are selected once from them; the
        leaves' pages are merged on the device (TopDocs.merge). Returns what the single-image method returns."""
        carr, ncl, qarr, nq = compile_queries(_resolve_all(queries, self))
        k = collector.num_hits_to_collect
        out = BatchResult(np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
                          np.zeros(nq, np.uint8))
        if _has_filter(additional):
            fr = _FilteredRecords(nq, _resolve_all(additional, self), lambda fields: (C.c_void_p * len(self.leaves))(
                *[l.sort_order(fields, stream).value for l in self.leaves]))
            check(self._lib.nrtgpu_searcher_search_bool_aggs_sorted_hits(self.handle, carr, ncl, qarr, nq, k, 0, *fr.sorted_args,
                                                                         C.c_void_p(stream), out.docs.ctypes.data,
                                                                         out.scores.ctypes.data, out.counts.ctypes.data,
                                                                         out.total_hits.ctypes.data))
            _keyword_keys(additional, fr.outs, self.keyword_term, self.keyword_names)
            return out, fr.outs
        aggs, res, narr, nres, n_nested, outs = _collector_records(nq, additional)
        check(self._lib.nrtgpu_searcher_search_bool_aggs_nested(self.handle, carr, ncl, qarr, nq, k, 0, aggs, len(additional), res,
                                                                narr, n_nested, nres, C.c_void_p(stream), out.docs.ctypes.data,
                                                                out.scores.ctypes.data, out.counts.ctypes.data,
                                                                out.total_hits.ctypes.data))
        _keyword_keys(additional, outs, self.keyword_term, self.keyword_names)
        return out, outs

    def search_tree_with_collectors(self, queries: Sequence[object], collector: RelevanceCollector, additional: Sequence[object],
                                    stream: int = 0):
        """GpuIndexSearcher.search_tree_with_collectors over the leaves (nrtgpu_searcher_search_tree_aggs), with the reader-wide
        tables and merges of search_with_collectors. Returns what the single-image method returns."""
        carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(_resolve_all(queries, self), phrase_table=True)
        k = collector.num_hits_to_collect
        out = BatchResult(np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
                          np.zeros(nq, np.uint8))
        fr = _FilteredRecords(nq, _resolve_all(additional, self), lambda fields: (C.c_void_p * len(self.leaves))(
            *[l.sort_order(fields, stream).value for l in self.leaves]))
        check(self._lib.nrtgpu_searcher_search_tree_aggs(self.handle, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, k, 0,
                                                         *fr.sorted_args, C.c_void_p(stream), out.docs.ctypes.data,
                                                         out.scores.ctypes.data, out.counts.ctypes.data, out.total_hits.ctypes.data))
        _keyword_keys(additional, fr.outs, self.keyword_term, self.keyword_names)
        return out, fr.outs

    def close(self):
        if self.handle:
            self._lib.nrtgpu_searcher_close(self.handle)
            self.handle = None


class GpuBatcher:
    """Request micro-batcher (nrtgpu_batcher_*): SearchHandler threads submit ONE query each and block; a native worker
    thread turns the waiting requests into batched nrtgpu_search_bool calls. The Java adaptor's counterpart is
    jni/java/.../GpuIndexSearcher.java (GpuBatcher.forIndex)."""

    def __init__(self, index: GpuIndex, max_batch: int = 256, max_wait_us: int = 200):
        self._lib = _native.gpu_lib()
        h = C.c_void_p()
        check(self._lib.nrtgpu_batcher_create(index.handle, max_batch, max_wait_us, C.byref(h)))
        self.handle, self.index = h, index

    def submit(self, query, collector: RelevanceCollector):
        """Blocking: returns (TopDocs, Diagnostics) of the one query."""
        carr, ncl, qarr, _ = compile_queries([_resolve_keywords(query, self.index)])
        k = collector.num_hits_to_collect
        docs, scores = np.zeros(k, np.int32), np.zeros(k, np.float32)
        cnt, tot, rel = C.c_int32(), C.c_int64(), C.c_uint8()
        diag = _native.Diagnostics()
        check(self._lib.nrtgpu_batcher_submit(self.handle, carr, ncl, qarr[0].min_should_match, k, collector.total_hits_threshold,
                                              docs.ctypes.data, scores.ctypes.data, C.byref(cnt), C.byref(tot), C.byref(rel), C.byref(diag)))
        n = cnt.value
        return TopDocs(TotalHits(tot.value, Relation(rel.value)), [ScoreDoc(int(d), float(s)) for d, s in zip(docs[:n], scores[:n])]), diag

    def stats(self):
        a, b = C.c_int64(), C.c_int64()
        check(self._lib.nrtgpu_batcher_stats(self.handle, C.byref(a), C.byref(b)))
        return {"batches": a.value, "requests": b.value}

    def close(self):
        if self.handle:
            self._lib.nrtgpu_batcher_close(self.handle)
            self.handle = None


NUM_CANDIDATES_LIMIT = 10000   # VectorFieldDef.java:74


@dataclass(frozen=True)
class KnnQuery:
    """KnnQuery of the search request as VectorFieldDef.getKnnQuery validates it (VectorFieldDef.java:401-425). The
    reference runs HNSW with a beam of num_candidates PER LEAF and merges the leaves' lists to k
    (NrtKnnFloatVectorQuery.java:43-64); here every leaf / shard is searched EXACTLY, so any num_candidates >= k yields the
    same -- exact -- top k (recall 1.0); it is validated and otherwise unused. similarity_threshold wraps the query in
    MinThresholdQuery(score >= similarityToScore(threshold)) (:590-593)."""
    k: int
    num_candidates: int
    similarity_threshold: Optional[float] = None

    def validate(self):
        if self.k < 1:
            raise ValueError("Vector search k must be >= 1")
        if self.num_candidates < self.k:
            raise ValueError("Vector search numCandidates must be >= k")
        if self.num_candidates > NUM_CANDIDATES_LIMIT:
            raise ValueError(f"Vector search numCandidates > {NUM_CANDIDATES_LIMIT}")


def similarity_to_score(similarity: float, sim: int, dims: int = 0, byte_field: bool = False) -> np.float32:
    """VectorFieldDef.similarityToScore (float :664-673, byte :870-881), float arithmetic."""
    s = np.float32(similarity)
    if sim == 0:
        return np.float32(1.0) / (np.float32(1.0) + s * s)
    if sim == 1 and byte_field:
        return np.float32(0.5) + s / np.float32(dims * (1 << 15))
    if sim in (1, 2):
        return (np.float32(1.0) + s) / np.float32(2.0)
    return np.float32(1.0) / (np.float32(1.0) + np.float32(-1.0) * s) if s < 0 else s + np.float32(1.0)


def normalized_cosine_vectors(vectors: np.ndarray):
    """What a `normalized_cosine` vector field does to its input (VectorFieldDef.java:308-332, 507-513, 568-573, 651-655):
    magnitude = sqrt(float dot(v, v)); v /= magnitude (float); the field is then searched with DOT_PRODUCT and the magnitude is
    kept in the <field>._magnitude float doc value. Returns (unit vectors float32, magnitudes float32)."""
    v = np.ascontiguousarray(vectors, np.float32)
    mag = np.sqrt(np.einsum("ij,ij->i", v, v, dtype=np.float32)).astype(np.float32)
    if (mag == 0).any():
        raise ValueError("Vector magnitude cannot be 0 when using cosine similarity")   # validateVectorForSearch :634-639
    return (v / mag[:, None]).astype(np.float32), mag


def blend_rrf(ctx: GpuContext, docs: np.ndarray, counts: np.ndarray, boosts: Sequence[float], rank_constant: int,
              top_hits: int):
    """BlenderOperation.blend with the weighted-RRF operation (BlenderOperation.java:76-87) for nq queries:
    docs [R, nq, top_in], counts [R, nq] -> (docs [nq, top_hits], scores, counts, total)."""
    d = np.ascontiguousarray(docs, np.int32)
    c = np.ascontiguousarray(counts, np.int32)
    b = np.ascontiguousarray(boosts, np.float32)
    R, nq, top_in = d.shape
    od, os_ = np.zeros((nq, top_hits), np.int32), np.zeros((nq, top_hits), np.float32)
    oc, ot = np.zeros(nq, np.int32), np.zeros(nq, np.int32)
    check(_native.gpu_lib().nrtgpu_blend_rrf(ctx.handle, R, nq, top_in, d.ctypes.data, c.ctypes.data, b.ctypes.data,
                                             rank_constant, top_hits, od.ctypes.data, os_.ctypes.data, oc.ctypes.data,
                                             ot.ctypes.data))
    return od, os_, oc, ot


def blend_scores(ctx: GpuContext, mode: str, docs: np.ndarray, scores: np.ndarray, counts: np.ndarray, boosts: Sequence[float],
                 top_hits: int):
    """BlenderOperation.blend with WeightedScoreOrderBlenderOperation (MAX / SUM / AVG of score * boost): docs, scores
    [R, nq, top_in], counts [R, nq] -> (docs [nq, top_hits], scores, counts, total)."""
    d = np.ascontiguousarray(docs, np.int32)
    s = np.ascontiguousarray(scores, np.float32)
    c = np.ascontiguousarray(counts, np.int32)
    b = np.ascontiguousarray(boosts, np.float32)
    R, nq, top_in = d.shape
    od, os_ = np.zeros((nq, top_hits), np.int32), np.zeros((nq, top_hits), np.float32)
    oc, ot = np.zeros(nq, np.int32), np.zeros(nq, np.int32)
    check(_native.gpu_lib().nrtgpu_blend_scores(ctx.handle, {"max": 1, "sum": 2, "avg": 3}[mode.lower()], R, nq, top_in, d.ctypes.data,
                                                s.ctypes.data, c.ctypes.data, b.ctypes.data, top_hits, od.ctypes.data, os_.ctypes.data,
                                                oc.ctypes.data, ot.ctypes.data))
    return od, os_, oc, ot


def rescore_combine(ctx: GpuContext, docs: np.ndarray, scores: np.ndarray, second_matches: np.ndarray,
                    second_scores: np.ndarray, query_weight: float, rescore_weight: float, counts=None):
    """QueryRescore (QueryRescore.java:39-57) for nq hit lists [nq, n_hits]: combined + re-sorted copies."""
    d = np.ascontiguousarray(docs, np.int32).copy()
    s = np.ascontiguousarray(scores, np.float32).copy()
    m = np.ascontiguousarray(second_matches, np.uint8)
    s2 = np.ascontiguousarray(second_scores, np.float32)
    nq, n_hits = d.shape
    cn = None if counts is None else np.ascontiguousarray(counts, np.int32)
    check(_native.gpu_lib().nrtgpu_rescore_combine(ctx.handle, nq, n_hits, None if cn is None else cn.ctypes.data,
                                                   d.ctypes.data, s.ctypes.data, m.ctypes.data, s2.ctypes.data,
                                                   query_weight, rescore_weight))
    return d, s
