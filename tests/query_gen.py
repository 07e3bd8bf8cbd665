"""Seeded random queries over the space the GPU engines support, each tagged with the engines that accept it. TEST
INFRASTRUCTURE ONLY.

Shapes: depth <= 4 (the root counts), <= 8 term slots (term leaves and phrase terms), <= 8 nested nodes, <= 32 clauses
(a phrase of n >= 2 terms adds n), every occur, msm from 0 to #SHOULD + 1, DisjunctionMaxQuery ties {0, 0.3, 1}.
Leaves: terms (absent, rare, mid, served by a tf plane, tf >= 255, on the second field, the same term twice), numeric
ranges (single- and multi-valued, lower > upper, int64 extremes), keyword ranges and prefixes, match-all, exact and
sloppy phrases of distinct terms. Boosts from BOOSTS on leaves, nodes and the root, up to three nested BoostQuerys on
one path; NESTED_BOOSTS is a triple whose float product depends on the order it is folded in.

Engine tags (engines()):
  - "flat_narrow": a flat BooleanQuery (or a bare leaf) of <= 16 clauses and <= 4 term clauses: the probe kernel;
  - "flat_wide":   a flat one of <= 8 term clauses: the window engine's flat instantiation (and the micro-batcher);
  - "tree":        every generated query: the window engine's tree instantiation."""
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, KeywordPrefixQuery, KeywordRangeQuery,
                                   MatchAllDocsQuery, Occur, PhraseQuery, RangeQuery, TermQuery)

BOOSTS = (0.0, 2.0**-149, 0.1, 0.5, 1.0, 1.75, 3.25, 1e6)
NESTED_BOOSTS = (0.1, 1.75, 3.25)   # outermost first: float32 products differ with the folding order
TIES = (0.0, 0.3, 1.0)
I64_MIN, I64_MAX = -(2**63), 2**63 - 1
MAX_DEPTH, MAX_SLOTS, MAX_NODES, MAX_CLAUSES = 4, 8, 8, 32
FLAT_MAX_CLAUSES = 16


@dataclass
class Space:
    """What the generator draws from, taken from one shard: term ids per category (TERM_KINDS and any other), phrase terms
    (field 0, with positions), numeric columns (index, multi-valued, (min, max) of the values) and keyword columns
    (index, sorted dictionary terms)."""
    terms: Dict[str, np.ndarray]
    phrase_terms: Optional[np.ndarray] = None
    columns: List[tuple] = field(default_factory=list)
    keyword: List[tuple] = field(default_factory=list)


TERM_KINDS = ("absent", "rare", "mid", "plane", "tf255", "field1")


class _Budget:
    def __init__(self):
        self.slots, self.nodes, self.clauses = 0, 0, 0


class Generator:
    def __init__(self, space: Space, seed: int):
        self.s, self.rng, self.seed = space, np.random.default_rng(seed), seed

    # ---------------------------------------------------------------- leaves

    def term(self, used: list) -> TermQuery:
        if used and self.rng.random() < 0.12:   # the same term twice in one query
            return TermQuery(int(used[self.rng.integers(len(used))]))
        kinds = [k for k in self.s.terms if len(self.s.terms[k])]
        pool = self.s.terms[kinds[self.rng.integers(len(kinds))]]
        t = int(pool[self.rng.integers(len(pool))])
        used.append(t)
        return TermQuery(t)

    def range_(self) -> RangeQuery:
        col, _, (lo, hi) = self.s.columns[self.rng.integers(len(self.s.columns))]
        r = self.rng.random()
        a, b = sorted(int(x) for x in self.rng.integers(lo, hi + 1, 2))
        if r < 0.1:
            return RangeQuery(col, b + 1, a)              # lower > upper: nothing
        if r < 0.2:
            return RangeQuery(col, I64_MIN, I64_MAX)
        if r < 0.3:
            return RangeQuery(col, I64_MIN, a)
        if r < 0.4:
            return RangeQuery(col, b, I64_MAX)
        return RangeQuery(col, a, b)

    def keyword(self):
        col, terms = self.s.keyword[self.rng.integers(len(self.s.keyword))]
        pick = lambda: terms[self.rng.integers(len(terms))]   # noqa: E731
        if self.rng.random() < 0.35:
            t = pick()
            cut = int(self.rng.integers(0, len(t) + 1))
            return KeywordPrefixQuery(col, t[:cut] if self.rng.random() < 0.85 else t + b"\x00")
        lo, hi = pick(), pick()
        if self.rng.random() < 0.7 and lo > hi:
            lo, hi = hi, lo
        if self.rng.random() < 0.2:
            lo = lo[:-1] + bytes([(lo[-1] + 1) % 256]) if lo else b"\x01"   # a bound the dictionary may not hold
        return KeywordRangeQuery(col, None if self.rng.random() < 0.15 else lo, None if self.rng.random() < 0.15 else hi,
                                 bool(self.rng.random() < 0.7), bool(self.rng.random() < 0.7))

    def phrase(self, n_terms: int) -> PhraseQuery:
        pool = self.s.phrase_terms
        terms = [int(x) for x in self.rng.choice(pool, n_terms, replace=False)]
        positions = None
        if self.rng.random() < 0.3:
            positions = sorted(int(x) for x in self.rng.choice(4, n_terms, replace=False))
        slop = 0 if self.rng.random() < 0.5 else int(self.rng.integers(1, 4))
        return PhraseQuery(terms, positions, slop)

    def boosted(self, q, root=False):
        r = self.rng.random()
        if r < 0.06:
            for b in reversed(NESTED_BOOSTS):
                q = BoostQuery(q, b)
            return q
        if r < (0.4 if root else 0.3):
            for _ in range(int(self.rng.integers(1, 4))):
                q = BoostQuery(q, BOOSTS[self.rng.integers(len(BOOSTS))] if self.rng.random() < 0.8 else 1.0)
        return q

    def leaf(self, bud: _Budget, used: list, tree: bool):
        r = self.rng.random()
        if self.s.phrase_terms is not None and tree and r < 0.12:
            n = int(self.rng.integers(1, 4))
            if bud.slots + n <= MAX_SLOTS and bud.clauses + 1 + (n if n > 1 else 0) <= MAX_CLAUSES:
                bud.slots += n
                bud.clauses += 1 + (n if n > 1 else 0)
                return self.boosted(self.phrase(n))
        bud.clauses += 1
        if r < 0.6 and bud.slots < MAX_SLOTS:
            bud.slots += 1
            return self.boosted(self.term(used))
        if r < 0.75 and self.s.columns:
            return self.boosted(self.range_())
        if r < 0.9 and self.s.keyword:
            return self.boosted(self.keyword())
        return self.boosted(MatchAllDocsQuery())

    # ---------------------------------------------------------------- nodes

    def node(self, depth: int, bud: _Budget, used: list, dismax: bool):
        n = int(self.rng.integers(1, 6))
        children = []
        for _ in range(n):
            if bud.clauses >= MAX_CLAUSES:
                break
            if depth < MAX_DEPTH and bud.nodes < MAX_NODES and self.rng.random() < 0.3:
                bud.nodes += 1
                bud.clauses += 1
                sub = self.boosted(self.node(depth + 1, bud, used, self.rng.random() < 0.35))
            else:
                sub = self.leaf(bud, used, True)
            children.append(sub)
        if dismax:
            return DisjunctionMaxQuery(children, TIES[self.rng.integers(len(TIES))])
        return self._bool(children)

    def _bool(self, children):
        occurs = [Occur(int(x)) for x in self.rng.choice(4, len(children), p=[0.45, 0.25, 0.15, 0.15])]
        n_should = sum(o == Occur.SHOULD for o in occurs)
        msm = int(self.rng.integers(0, n_should + 2)) if self.rng.random() < 0.35 else 0
        q = BooleanQuery(minimum_number_should_match=msm)
        for c, o in zip(children, occurs):
            q.add(c, o)
        return q

    def tree_query(self):
        bud = _Budget()
        used = []
        if self.rng.random() < 0.1:   # a bare leaf or dismax at the root
            if self.rng.random() < 0.5:
                bud.nodes += 1
                bud.clauses += 1
                return self.boosted(self.node(2, bud, used, True), root=True)
            return self.boosted(self.leaf(bud, used, True), root=True)
        return self.boosted(self.node(1, bud, used, False), root=True)

    def flat_query(self, max_terms: int):
        bud = _Budget()
        used = []
        n = int(self.rng.integers(1, FLAT_MAX_CLAUSES + 1)) if self.rng.random() < 0.2 else int(self.rng.integers(1, 7))
        children, n_terms = [], 0
        for _ in range(n):
            c = self.leaf(bud, used, False)
            inner = c
            while isinstance(inner, BoostQuery):
                inner = inner.query
            if isinstance(inner, TermQuery):
                if n_terms == max_terms:
                    continue
                n_terms += 1
            children.append(c)
        if len(children) == 1 and self.rng.random() < 0.3:
            return self.boosted(children[0], root=True)
        return self.boosted(self._bool(children), root=True)

    def query(self):
        r = self.rng.random()
        if r < 0.25:
            return self.flat_query(4)
        if r < 0.4:
            return self.flat_query(8)
        return self.tree_query()

    def queries(self, n: int):
        return [self.query() for _ in range(n)]


def space_of(sh, columns, plane_terms=None, phrase_terms=None) -> Space:
    """The Space of HostShard sh: term categories from its lists (plane: plane_terms, else the 8 longest field-0 lists),
    the numeric columns given as (index, multi_valued) with their value bounds, every keyword column, and phrase_terms
    (or none when sh has no positions)."""
    df = np.diff(sh.term_off)
    tf = np.zeros(len(df), np.int64)
    owner = np.repeat(np.arange(len(df)), df)
    np.maximum.at(tf, owner, sh.post_freqs)
    fld = np.zeros(len(df), np.int32) if sh.term_field is None else np.asarray(sh.term_field)
    f0 = np.nonzero((fld == 0) & (df > 0) & (tf < 255))[0]
    by_df = f0[np.argsort(df[f0], kind="stable")]
    terms = {"absent": np.nonzero(df == 0)[0], "tf255": np.nonzero(tf >= 255)[0],
             "field1": np.nonzero((fld == 1) & (df > 0))[0],
             "rare": by_df[:max(1, len(by_df) // 5)], "mid": by_df[len(by_df) * 2 // 5:len(by_df) * 4 // 5],
             "plane": by_df[-8:] if plane_terms is None else np.asarray(plane_terms)}
    cols = []
    for c, multi in columns:
        v = np.asarray(sh.columns[c])
        cols.append((c, multi, (int(v.min()) - 2, int(v.max()) + 2)))
    kw = [(k, [bytes(t) for t in col.terms]) for k, col in enumerate(sh.keyword_columns) if len(col.terms)]
    if sh.post_positions is None:
        phrase_terms = None
    return Space(terms, None if phrase_terms is None else np.asarray(phrase_terms), cols, kw)


def _unboost(q):
    while isinstance(q, BoostQuery):
        q = q.query
    return q


def engines(q) -> set:
    """the engine tags of query object q (module docstring)"""
    root = _unboost(q)
    clauses = [c.query for c in root.clauses] if isinstance(root, BooleanQuery) else [root]
    leaves = [_unboost(c) for c in clauses]
    tags = {"tree"}
    if any(isinstance(x, (BooleanQuery, DisjunctionMaxQuery, PhraseQuery)) for x in leaves) or len(leaves) > FLAT_MAX_CLAUSES:
        return tags
    n_terms = sum(isinstance(x, TermQuery) for x in leaves)
    if n_terms <= 8:
        tags.add("flat_wide")
    if n_terms <= 4:
        tags.add("flat_narrow")
    return tags


def describe(seed: int, i: int, q) -> str:
    """what a failure prints: the seed, the query's index in the batch and its repr"""
    return f"seed {seed} query {i}: {q!r}"
