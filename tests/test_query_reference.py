"""The object-level reference (tests/query_reference.py) on the CPU: pinned to the known answers of the reference's own
tests, then compared, over a few hundred generated queries (tests/query_gen.py) on small seeded shards, with the judges
the GPU suites use -- oracle.search_compiled over compile_queries for flat queries, phrase_reference / tree_reference over
compile_tree for every query. The two sides share no code but the query objects, so this puts the Python query compilers
under test: boost folding, node numbering, msm and tie breakers on the right nodes, every clause kept."""
import numpy as np
import pytest

import oracle
import phrase_reference as pr
import query_gen as qg
from helpers import shard_from_token_docs
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, KeywordPrefixQuery, KeywordRangeQuery,
                                   MatchAllDocsQuery, Occur, PhraseQuery, RangeQuery, ScoreDoc, TermQuery, compile_queries)
from query_reference import Reference, bm25, byte4_to_int, idf, length_cache

import keyword_query_reference as kqr

S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT


def f32(x):
    return float(np.float32(x))


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(c, o)
    return q


# ---------------------------------------------------------------- known answers (tests/test_oracle_golden.py)

def scores_of(sh, q, k=10):
    d, s, c, t = Reference(sh).search([q], k)
    return d[0, :c[0]].tolist(), s[0, :c[0]], int(t[0])


def test_smallfloat_and_bm25_constants():
    assert [byte4_to_int(oracle.int_to_byte4(i)) for i in (40, 41, 100, 1000)] == [40, 40, 96, 984]
    assert all(byte4_to_int(b) == oracle.byte4_to_int(b) for b in range(256))
    assert f32(idf(1, 2)) == f32(0.6931472) and f32(idf(2, 2)) == f32(0.18232156)
    cache = length_cache(1.2, 0.75, np.float32(4.0))   # QueryTest.java:1003-1018: tf = 0.45454544 at dl = avgdl = 4
    one, norm = np.ones(1, np.int32), np.array([oracle.int_to_byte4(4)])
    assert abs(float(bm25(np.float32(1), one, norm, cache)[0]) - 0.45454544) < 1e-7
    idf_sum = np.float32(float(idf(1, 2)) + float(idf(2, 2)))
    assert f32(idf_sum) == f32(0.87546873) and f32(bm25(idf_sum, one, norm, cache)[0]) == f32(0.3979403)


def test_known_term_scores():
    # MultiFunctionScoreQueryTest: text_field:"Document2" -> docs 2, 4 at 0.33812057971954346 / 0.27725890278816223
    docs = ["Document1 with none of filter terms", "Document2 with term1 filter term",
            "Document1 with term2 filter term", "Document2 with both term1 and term2 filter terms"]
    sh, v = shard_from_token_docs([[d.lower().split() for d in docs]])
    d, s, t = scores_of(sh, TermQuery(v[(0, "document2")]))
    assert d == [1, 3] and t == 2 and float(s[0]) == 0.33812057971954346 and float(s[1]) == 0.27725890278816223
    # SearchStateTest: vendor over {"first vendor", "second vendor review"}: doc 1 scores 0.0766057
    sh, v = shard_from_token_docs([["first vendor".split(), "second vendor review".split()]])
    d, s, t = scores_of(sh, TermQuery(v[(0, "vendor")]))
    assert d == [0, 1] and abs(float(s[1]) - 0.0766057) < 1e-7
    # docker-compose search.json: first SHOULD vendor SHOULD -> 0.3979403 (summed in double), 0.0828734
    sh, v = shard_from_token_docs([["first vendor".split(), "second vendor".split()]])
    d, s, t = scores_of(sh, bq((TermQuery(v[(0, "first")]), S), (TermQuery(v[(0, "vendor")]), S)))
    assert d == [0, 1] and t == 2 and f32(s[0]) == f32(0.3979403) and abs(float(s[1]) - 0.0828734) < 1e-7
    # SimilarityTest: bm25(first, tf = 2) = 0.43321696
    sh, v = shard_from_token_docs([[["first", "vendor", "first", "again"], ["second", "vendor", "second", "again"]]])
    assert abs(float(scores_of(sh, TermQuery(v[(0, "first")]))[1][0]) - 0.43321696) < 1e-7


def test_known_phrase_score():
    # QueryTest.java:1003-1018: the phrase "first vendor" at dl = avgdl = 4: idf sum 0.87546873, score 0.3979403
    sh = pr.shard_from_tokens([[[[0, 1, 2, 3]]], [[[4, 1, 2, 3]]]], [0] * 5, 1)
    d, s, t = scores_of(sh, PhraseQuery([0, 1]))
    assert d == [0] and t == 1 and f32(s[0]) == f32(0.3979403)


def test_known_boost_ranges_match_all_and_paging():
    sh, v = shard_from_token_docs([["first vendor".split(), "second vendor review".split()]],
                                  columns=[np.array([3, 7], np.int64), np.array([12, 16], np.int64)])
    t = TermQuery(v[(0, "vendor")])
    assert np.array_equal(scores_of(sh, t)[1] * np.float32(2), scores_of(sh, BoostQuery(t, 2.0))[1])
    for col, lo, hi in ((0, 5, 10), (1, 15, 19)):    # QueryTest.testSearchRangeQuery: doc "2" only, constant score 1
        d, s, n = scores_of(sh, RangeQuery(col, lo, hi))
        assert d == [1] and n == 1 and float(s[0]) == 1.0
    d, s, n = scores_of(sh, MatchAllDocsQuery())
    assert d == [0, 1] and all(float(x) == 1.0 for x in s)
    # IntFieldDefTest multi_stored: {MIN_VALUE, 15}, {1, 15}, no value
    imin = -(2**31)
    sh, _ = shard_from_token_docs([[["a"], ["a"], ["a"]]], columns=[np.array([imin, 15, 1, 15], np.int64)])
    sh.column_offsets = [np.array([0, 2, 4, 4], np.int64)]
    for lo, hi, want in ((15, 15, [0, 1]), (0, 10, [1]), (imin, imin, [0]), (2, 14, []), (imin, 2**31 - 1, [0, 1])):
        assert scores_of(sh, RangeQuery(0, lo, hi))[0] == want
    # LazyQueueTopScoreDocCollector: ties by doc, searchAfter skips (score, doc) <= after; totalHits unchanged
    sh, v = shard_from_token_docs([[["x", "pad"]] * 6])
    r = Reference(sh)
    d, s, c, tot = r.search([TermQuery(v[(0, "x")])], 4)
    assert d[0].tolist() == [0, 1, 2, 3] and tot[0] == 6
    d2, s2, c2, tot2 = r.search([TermQuery(v[(0, "x")])], 4, [ScoreDoc(3, float(s[0, 3]))])
    assert c2[0] == 2 and d2[0, :2].tolist() == [4, 5] and tot2[0] == 6


# ---------------------------------------------------------------- generated queries against the compiled judges

def small_shard(seed: int, n_docs: int = 3000):
    """Two text fields with positions (field 1 without norms), terms with tf >= 255 and absent terms, a single-valued
    column with missing values, a multi-valued one, a SORTED and a SORTED_SET keyword column, and 5% deletes."""
    rng = np.random.default_rng(seed)
    v0, v1 = 200, 60
    doc, term, pos = [], [], []
    for f, (lo, mean, vocab, base) in enumerate(((3, 8.0, v0 - 3, 0), (1, 3.0, v1 - 1, v0))):
        lens = lo + rng.poisson(mean, n_docs)
        d = np.repeat(np.arange(n_docs), lens)
        t = base + np.minimum(rng.zipf(1.3, len(d)) - 1, vocab - 1)
        p = np.concatenate([rng.permutation(n) for n in lens])
        doc.append(d), term.append(t), pos.append(p)
    heavy = rng.choice(n_docs, 6, replace=False)      # term v0 - 1: tf 255 .. 400 in six docs
    for i, dd in enumerate(heavy):
        tf = 255 + 30 * i
        doc.append(np.full(tf, dd)), term.append(np.full(tf, v0 - 1)), pos.append(1000 + np.arange(tf))
    # terms v0 - 3, v0 - 2 (field 0) and v0 + v1 - 1 (field 1) hold no posting: df 0
    term_field = np.array([0] * v0 + [1] * v1, np.int32)
    sh = pr.shard_from_token_arrays(n_docs, term_field, 2, np.concatenate(doc), np.concatenate(term), np.concatenate(pos))
    sh.fields[1].norms = None
    has = (rng.random(n_docs) < 0.9).astype(np.uint8)
    cnt = rng.integers(0, 4, n_docs)
    moff = np.zeros(n_docs + 1, np.int64)
    np.cumsum(cnt, out=moff[1:])
    mv = rng.integers(0, 200, int(moff[-1])).astype(np.int64)
    mv = mv[np.lexsort((mv, np.repeat(np.arange(n_docs), cnt)))]
    sh.columns = [rng.integers(-1000, 1001, n_docs).astype(np.int64), mv]
    sh.column_has = [has, None]
    sh.column_offsets = [None, moff]
    words = ["", "a", "ab", "abc", "abd", "b", "ba", "bz", "café", "cafe", "d\U0001F600", "zz", "zza"]
    one = [None if rng.random() < 0.1 else words[rng.integers(len(words))] for _ in range(n_docs)]
    many = [[words[i] for i in rng.choice(len(words), rng.integers(0, 4), replace=False)] for _ in range(n_docs)]
    sh.keyword_columns = [ix.KeywordColumn.from_values(one, False), ix.KeywordColumn.from_values(many, True)]
    sh.live_docs = (rng.random(n_docs) > 0.05).astype(np.uint8)
    return sh


def with_shadow_columns(sh):
    """sh plus, for each keyword column k, numeric column 2 + k holding the codes 2i + 2 of its terms (multi-valued for
    SORTED_SET): what a keyword clause means to the judges that only know numeric ranges"""
    cols, has, offs = list(sh.columns), list(sh.column_has), list(sh.column_offsets)
    for col in sh.keyword_columns:
        codes = 2 * np.asarray(col.ords, np.int64) + 2
        if col.multi_valued:
            cols.append(codes), has.append(None), offs.append(np.asarray(col.offsets, np.int64))
        else:
            cols.append(np.where(codes > 0, codes, 0)), has.append((codes > 0).astype(np.uint8)), offs.append(None)
    out = ix.HostShard(**{**sh.__dict__, "columns": cols, "column_has": has, "column_offsets": offs})
    return out


def shadow(q, sh):
    """q with every keyword leaf replaced by the code range of its shadow column; the matched terms of a keyword range
    are one run of the dictionary, asserted here"""
    if isinstance(q, (KeywordRangeQuery, KeywordPrefixQuery)):
        col = sh.keyword_columns[q.column]
        if isinstance(q, KeywordPrefixQuery):
            pred = kqr.prefix_pred(q.prefix)
        else:
            pred = kqr.range_pred(q.lower, q.upper, q.include_lower, q.include_upper)
        hit = np.nonzero([pred(bytes(t)) for t in col.terms])[0]
        if len(hit) == 0:
            return RangeQuery(2 + q.column, 1, 0)
        assert hit[-1] - hit[0] + 1 == len(hit)
        return RangeQuery(2 + q.column, 2 * int(hit[0]) + 2, 2 * int(hit[-1]) + 2)
    if isinstance(q, BoostQuery):
        return BoostQuery(shadow(q.query, sh), q.boost)
    if isinstance(q, BooleanQuery):
        return BooleanQuery([type(c)(shadow(c.query, sh), c.occur) for c in q.clauses], q.minimum_number_should_match)
    if isinstance(q, DisjunctionMaxQuery):
        return DisjunctionMaxQuery([shadow(d, sh) for d in q.disjuncts], q.tie_breaker)
    return q


def same_pages(got, want, k, queries, seed, what):
    for i in range(len(queries)):
        n = int(want[2][i])
        msg = f"{what}: {qg.describe(seed, i, queries[i])}"
        assert int(got[2][i]) == n, f"{msg}: counts {got[2][i]} vs {n}"
        assert np.array_equal(got[0][i, :n], want[0][i, :n]), f"{msg}: docs differ"
        assert np.array_equal(got[1][i, :n].view(np.uint32), want[1][i, :n].view(np.uint32)), f"{msg}: scores differ"
        assert int(got[3][i]) == int(want[3][i]), f"{msg}: totalHits {got[3][i]} vs {want[3][i]}"


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generated_queries_equal_the_compiled_judges(built, seed):
    sh = small_shard(seed)
    judge_sh = with_shadow_columns(sh)
    space = qg.space_of(sh, [(0, False), (1, True)], phrase_terms=np.arange(0, 40))
    gen = qg.Generator(space, seed)
    queries = gen.queries(150)
    ref = Reference(sh)
    k = 50
    want = ref.search(queries, k)
    assert (want[3] > 0).mean() > 0.35 and (want[3] > k).any()
    shadowed = [shadow(q, sh) for q in queries]
    oix = oracle.OracleIndex(judge_sh)
    tree = pr.search(judge_sh, shadowed, k, oix=oix)
    same_pages(tree, want, k, queries, seed, "compile_tree + phrase_reference")
    flat = [i for i, q in enumerate(queries) if "flat_wide" in qg.engines(q)]
    assert len(flat) > 20
    carr, ncl, qarr, nq = compile_queries([shadowed[i] for i in flat])
    got = oracle.search_compiled(oix, carr, ncl, qarr, nq, k)
    same_pages(got, [w[flat] for w in want], k, [queries[i] for i in flat], seed, "compile_queries + oracle")
    # searchAfter from the reference's own pages
    rng = np.random.default_rng(seed)
    after = []
    for i in range(len(queries)):
        n = int(want[2][i])
        if n == 0:
            after.append(None)
            continue
        r = int(rng.integers(n))
        after.append(ScoreDoc(int(want[0][i, r]), float(want[1][i, r])))
    want2 = ref.search(queries, k, after)
    tree2 = pr.search(judge_sh, shadowed, k, search_after=after, oix=oix)
    same_pages(tree2, want2, k, queries, seed, "compile_tree + phrase_reference, searchAfter")


def test_generator_covers_the_space(built):
    sh = small_shard(1)
    space = qg.space_of(sh, [(0, False), (1, True)], phrase_terms=np.arange(0, 40))
    queries = qg.Generator(space, 7).queries(400)
    seen = set()

    def walk(q, depth):
        nb = 0
        while isinstance(q, BoostQuery):
            seen.add(("boost", q.boost))
            nb += 1
            q = q.query
        seen.add(("nested boosts", nb))
        if isinstance(q, BooleanQuery):
            seen.add(("depth", depth))
            seen.add(("msm above #SHOULD", q.minimum_number_should_match > sum(c.occur == S for c in q.clauses)))
            for c in q.clauses:
                seen.add(("occur", c.occur))
                walk(c.query, depth + 1)
        elif isinstance(q, DisjunctionMaxQuery):
            seen.add(("tie", q.tie_breaker))
            for d in q.disjuncts:
                walk(d, depth + 1)
        else:
            seen.add(type(q).__name__)
            if isinstance(q, PhraseQuery):
                seen.add(("slop", q.slop > 0))
            if isinstance(q, RangeQuery):
                seen.add(("range", q.column, q.lower > q.upper, q.lower == qg.I64_MIN or q.upper == qg.I64_MAX))
            if isinstance(q, TermQuery):
                for kind, pool in space.terms.items():
                    if q.term in pool:
                        seen.add(("term", kind))

    for q in queries:
        walk(q, 1)
    want = {("boost", b) for b in qg.BOOSTS} | {("depth", d) for d in (1, 2, 3, 4)} | {("occur", o) for o in Occur}
    want |= {("tie", t) for t in qg.TIES} | {("term", k) for k in qg.TERM_KINDS} | {("nested boosts", 3), ("slop", True), ("slop", False)}
    want |= {("msm above #SHOULD", True)} | {("range", c, x, y) for c in (0, 1) for x in (False, True) for y in (False, True) if not (x and y)}
    want |= {"PhraseQuery", "KeywordRangeQuery", "KeywordPrefixQuery", "MatchAllDocsQuery"}
    assert want <= seen, sorted(map(str, want - seen))
    tags = [qg.engines(q) for q in queries]
    assert sum("flat_narrow" in t for t in tags) > 50 and sum(t == {"tree"} for t in tags) > 150
