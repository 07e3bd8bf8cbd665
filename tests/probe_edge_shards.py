"""Shards built in numpy whose posting lists sit on the structural edges of posting_probe_kernel (probe_kernel.cuh) and
its work planner (batch_plan.inc), and the query batches that reach them. Shared by tests/test_probe_edges_plan.py (the
plan-side facts, on the CPU) and tests/test_gpu_probe_edges.py (oracle parity and the kernel's own counters).

Edge shard: 1,250,003 docs (n mod 4 = 3: the 2-bit plane's tail byte is partial; n mod 1024 = 723: the last granule is
partial), so the planner cuts 3 slices of 407 granules; a query of > 1.57M postings is split into 16 parts of
fine = ceil(407 / 16) = 26 granules, fewer than the 32 warm-up granules (kWarmGran).
Small shard: 200,003 docs (< 262,144): lists of df >= n / 64 get a tf plane, but only lists of df >= 4096 get a
granule row, so the lists of df 3126..4095 are planes without skip data."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np

import oracle
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import BooleanQuery, MatchAllDocsQuery, Occur, RangeQuery, TermQuery

N_EDGE = 1_250_003
N_SMALL = 200_003
GRAN = 1024
SLICE_DOCS = 407 * GRAN                      # the planner's slice of the edge shard (3 slices)
K_SHORT_MAX = {"A": 8192 - 4 * 1056, "B": 6656 - 4 * 1056}   # kStage - kLongReserve of the two stage configurations
CLUSTER_GRANS = list(range(24, 34)) + list(range(405, 410)) + [1218, 1219, 1220]   # part 0/1 edge, slice 0/1 edge, the tail
NMIN_LEN = 2                                 # the shortest field-0 length (held by docs of T_TIGHT only)
TIE_STRIDE = 216
TFS = np.array([1, 2, 3, 254, 255, 256, 300, 4], np.int32)   # every tf class: 2-bit codes 1..3, the 254/255 byte edge, > 255
_BYTE4 = np.array([oracle.int_to_byte4(n) for n in range(1024)], np.uint8)


@dataclass
class Built:
    shard: ix.HostShard
    term: Dict[str, int]                                   # list name -> term id
    post_base: Dict[str, int] = field(default_factory=dict)


def _spread(lo: int, hi: int, n: int) -> np.ndarray:
    """n distinct docs spread evenly over [lo, hi), both ends included."""
    d = np.unique(np.linspace(lo, hi - 1, n).round().astype(np.int64))
    assert len(d) == n, (lo, hi, n)
    return d


def _tf_cycle(docs: np.ndarray, salt: int) -> np.ndarray:
    """every tf class in turn along the list (5 is coprime with the 8 classes)"""
    return TFS[(np.arange(len(docs)) * 5 + salt) % len(TFS)]


class _Image:
    """Posting lists in image order; a list may ask for its first posting at a given residue mod 16 (a filler list of
    1..15 postings is inserted before it)."""

    def __init__(self):
        self.lists: List = []        # (name, docs, tfs, field)
        self.n = 0

    def add(self, name, docs, tfs, fld=0, pbm=None):
        docs = np.asarray(docs, np.int64)
        assert (np.diff(docs) > 0).all()
        if pbm is not None and self.n % 16 != pbm:
            k = (pbm - self.n) % 16
            self.lists.append((f"_fill{len(self.lists)}", np.arange(k, dtype=np.int64) * 97 + 5, np.ones(k, np.int32), fld))
            self.n += k
        self.lists.append((name, docs, np.asarray(tfs, np.int32), fld))
        self.n += len(docs)

    def shard(self, n_docs, fields, columns=()):
        off = np.zeros(len(self.lists) + 1, np.int64)
        off[1:] = np.cumsum([len(d) for _, d, _, _ in self.lists])
        sh = ix.HostShard(n_docs=n_docs, doc_base=0, term_off=off,
                          post_docs=np.concatenate([d for _, d, _, _ in self.lists]).astype(np.int32),
                          post_freqs=np.concatenate([f for _, _, f, _ in self.lists]).astype(np.int32),
                          fields=fields, term_field=np.array([f for _, _, _, f in self.lists], np.int32),
                          columns=list(columns), column_has=[None] * len(columns))
        sh.term_df = np.diff(off).astype(np.int64)
        term = {name: i for i, (name, _, _, _) in enumerate(self.lists)}
        return Built(sh, term, {name: int(off[i]) for name, i in term.items()})


def edge_shard() -> Built:
    n = N_EDGE
    rng = np.random.default_rng(2024)
    im = _Image()
    alld = np.arange(n, dtype=np.int64)
    tie = np.arange(2000, dtype=np.int64) * TIE_STRIDE                      # 0 .. 431,784: parts 0-16 and the slice 0/1 edge
    tie_top = tie[::100] + TIE_STRIDE // 2                                  # 20 docs that outscore the tie group (one tie of their own)
    plain = np.ones(n, bool)                                                # docs whose D0 / D1 tf stays 1 (tie docs score alike)
    plain[tie] = plain[tie_top] = False
    # D0: every doc (plane); D1: every second doc (plane); special tfs on a sparse comb away from the tie docs
    f0 = np.ones(n, np.int32)
    sp = (alld % 97 == 13) & plain
    f0[sp] = _tf_cycle(alld[sp], 0)
    im.add("D0", alld, f0)
    d1 = alld[::2]
    f1 = np.ones(len(d1), np.int32)
    sp1 = (d1 % 89 == 7) & plain[d1]
    f1[sp1] = _tf_cycle(d1[sp1], 3)
    im.add("D1", d1, f1)
    # the index-build rule edges: plane at df * 64 >= n, granule row at df >= 4096
    df_plane = -(-n // 64)
    for name, df in (("P_HI", df_plane), ("P_LO", df_plane - 1), ("G_HI", 4096), ("G_LO", 4095)):
        d = _spread(0, n, df)
        im.add(name, d, _tf_cycle(d, len(name)))
    # four clustered long lists (no plane, granule rows) filling the same granules: 4 x 1024 postings in a granule is the
    # long-list reserve of the stage, so runs shrink to one granule; the last doc of every granule has tf 3 or > 255
    cl = np.concatenate([np.arange(g * GRAN, min((g + 1) * GRAN, n)) for g in CLUSTER_GRANS]).astype(np.int64)
    for i in range(4):
        f = (1 + (cl * (i + 3)) % 2).astype(np.int32)
        last = (cl % GRAN == GRAN - 1) | (cl == n - 1)
        f[last] = 3 if i % 2 else 260 + i
        f[cl % GRAN == 0] = 2
        im.add(f"C{i}", cl, f)
    # a short list with postings in every granule of the clusters (narrowed in place, then from the staged copy)
    srun = cl[(cl * 7919) % 13 == 0]
    im.add("S_RUN", srun, _tf_cycle(srun, 1))
    # short lists at the staging limits (first posting 16-aligned: seg_n = the list length rounded up to 16), every posting
    # in slice 1 so one work item holds the whole list
    for L in (2431, 2432, 2433, 3967, 3968, 3969, 1216, 1232, 1984, 2000):
        d = _spread(SLICE_DOCS + 3, 2 * SLICE_DOCS - 5, L)
        im.add(f"SH_{L}", d, _tf_cycle(d, L), pbm=0)
        if L in (1216, 1984):
            d = _spread(SLICE_DOCS + 11, 2 * SLICE_DOCS - 17, L)
            im.add(f"SH_{L}b", d, _tf_cycle(d, L + 1), pbm=0)
    # the tie group (tf 1, one field length, tf 1 in D0 and D1: equal scores) spanning part and slice edges
    tdocs = np.union1d(tie, tie_top)
    im.add("T_TIE", tdocs, np.where(np.isin(tdocs, tie_top), 3, 1))
    # tight bounds: docs at the shortest field length with tf 1, 2, 3, 255 and > 255 (they reach the tf-pattern bound)
    tight = _spread(7, n - 7, 6000)
    ttf = np.where(np.arange(len(tight)) % 3 == 0, TFS[np.arange(len(tight)) % 8], 1).astype(np.int32)
    im.add("T_TIGHT", tight, ttf)
    # every granule edge, every slice edge, n - 1
    edges = np.unique(np.concatenate([np.arange(GRAN, n, GRAN) - 1, np.arange(GRAN, n, GRAN), [0, n - 1],
                                      np.arange(1, 3) * SLICE_DOCS - 1, np.arange(1, 3) * SLICE_DOCS]))
    im.add("E_EDGES", edges, _tf_cycle(edges, 5))
    # heavy query pieces: a rare list with a high bound (< 2 * top_k postings: a first-docs warm-up item) and a short list
    # in the granules a kItemBehindWarm part 1 starts behind (26..31) and around them
    rare = np.array([3, 1023, 1024, 26 * GRAN - 1, 26 * GRAN, 32 * GRAN - 1, 32 * GRAN, SLICE_DOCS - 1, SLICE_DOCS, n - 1] +
                    rng.choice(n, 20, replace=False).tolist())
    rare = np.unique(rare)
    im.add("R_RARE", rare, _tf_cycle(rare, 2))
    sw = np.unique(np.concatenate([np.arange(20 * GRAN, 40 * GRAN, 37), [26 * GRAN - 1, 26 * GRAN, 32 * GRAN - 1, 32 * GRAN]]))
    im.add("S_WARM", sw, _tf_cycle(sw, 4))
    # omitNorms field (field 1): a plane, a long list, a short list
    for name, m in (("O_PLANE", 40_000), ("O_LONG", 9_000), ("O_SHORT", 3_000)):
        d = np.sort(rng.choice(n, m, replace=False))
        im.add(name, d, _tf_cycle(d, m), fld=1)
    # 16 lists of 16 * 17 + 1 postings: their first postings take every residue mod 16; the last one ends the image
    for i in range(16):
        d = _spread(13 * i, n, 273)                                         # (n - 1 included)
        im.add(f"A{i}", d, _tf_cycle(d, i))
    # field lengths: 3..40 at random, the tight docs the shortest, the tie docs one length
    lens = rng.integers(3, 41, n)
    lens[tight[ttf > 1]] = NMIN_LEN
    lens[tight[::5]] = NMIN_LEN
    lens[tie] = 9
    lens[tie_top] = 9
    norms = _BYTE4[lens]
    col = ((alld * 2654435761) % 1000).astype(np.int64)
    b = im.shard(n, [ix.TextField(norms, n, int(lens.sum())), ix.TextField(None, n, 4 * n)], columns=[col])
    return b


def small_shard() -> Built:
    """200,003 docs: planes without granule rows (df 3126 and 4095), planes with rows, short lists, and a dense list."""
    n = N_SMALL
    rng = np.random.default_rng(7)
    im = _Image()
    for name, df in (("PL_MIN", -(-n // 64)), ("PL_NOROW", 4095), ("PL_ROW", 4096), ("DENSE", n // 3),
                     ("SHORT", 900), ("SHORT2", 2500), ("BELOW", -(-n // 64) - 1)):
        d = _spread(0, n, df) if name != "DENSE" else np.arange(0, n, 3)
        im.add(name, d, _tf_cycle(d, df))
    lens = rng.integers(2, 30, n)
    return im.shard(n, [ix.TextField(_BYTE4[lens], n, int(lens.sum()))], columns=[(np.arange(n) % 500).astype(np.int64)])


# ---------------------------------------------------------------- query batches

def disj(*terms):
    q = BooleanQuery()
    for t in terms:
        q.add(TermQuery(int(t)), Occur.SHOULD)
    return q


def bq(*clauses):
    q = BooleanQuery()
    for c, o in clauses:
        q.add(TermQuery(int(c)) if isinstance(c, (int, np.integer)) else c, o)
    return q


def edge_batches(b: Built) -> Dict[str, list]:
    t = b.term
    S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
    disjs = [disj(t["C0"], t["C1"], t["C2"], t["C3"]), disj(t["C0"], t["C1"], t["C2"], t["S_RUN"]),
             disj(t["C3"], t["C2"], t["C1"], t["SH_3969"]), disj(t["S_RUN"], t["C0"], t["C1"]),
             *[disj(t[f"SH_{L}"]) for L in (2431, 2432, 2433, 3967, 3968, 3969)],
             disj(t["SH_1216"], t["SH_1216b"]), disj(t["SH_1216"], t["SH_1232"]),
             disj(t["SH_1984"], t["SH_1984b"]), disj(t["SH_1984"], t["SH_2000"]),
             disj(t["P_HI"]), disj(t["P_LO"]), disj(t["P_HI"], t["P_LO"]), disj(t["G_HI"], t["G_LO"]),
             disj(t["G_LO"], t["P_HI"], t["C0"]),
             disj(t["T_TIGHT"]), disj(t["T_TIGHT"], t["P_HI"]), disj(t["D1"], t["T_TIGHT"]),
             disj(t["T_TIE"], t["D0"], t["D1"]), disj(t["S_WARM"], t["R_RARE"], t["D0"], t["D1"]),
             disj(t["E_EDGES"]), disj(t["E_EDGES"], t["C0"]), disj(t["E_EDGES"], t["D1"], t["G_HI"]),
             disj(t["R_RARE"], t["R_RARE"]), disj(t["P_HI"], t["G_LO"], t["P_HI"]),
             *[disj(t[f"A{i}"]) for i in range(16)], disj(t["A14"], t["A15"], t["C3"]), disj(t["A15"], t["A0"]),
             disj(t["O_PLANE"]), disj(t["O_SHORT"]), disj(t["O_PLANE"], t["O_SHORT"]),
             disj(t["O_LONG"], t["O_PLANE"], t["O_SHORT"], t["O_LONG"])]
    rng = RangeQuery(0, 100, 599)
    conj = [bq((t["C0"], M), (t["C1"], M)), bq((t["C0"], M), (t["C1"], S), (t["C2"], N)),
            bq((t["G_LO"], M), (rng, F), (t["P_HI"], S)), bq((t["T_TIGHT"], M), (t["E_EDGES"], N), (t["D1"], S)),
            bq((t["SH_3969"], M), (t["C0"], S)), bq((t["P_LO"], F), (t["P_HI"], M), (t["C3"], N)),
            bq((t["A15"], M), (t["A0"], S)), bq((t["C2"], M), (t["S_RUN"], M), (rng, F)),
            bq((t["D1"], M), (t["T_TIE"], M), (t["E_EDGES"], N)), bq((t["O_PLANE"], M), (t["O_SHORT"], S), (t["O_LONG"], N))]
    dense = [bq((rng, F), (t["C0"], S), (t["C1"], S)),
             bq((MatchAllDocsQuery(), M), (t["C0"], S), (t["C1"], S), (t["C2"], S), (t["C3"], S)),
             bq((MatchAllDocsQuery(), S), (t["T_TIGHT"], S)),
             bq((RangeQuery(0, 0, 999), F), (t["D1"], N), (t["E_EDGES"], S)),
             bq((rng, M), (t["S_RUN"], S), (t["A15"], S))]
    return {"disj": disjs, "conj": conj, "dense": dense}


def small_batches(b: Built) -> list:
    t = b.term
    return [disj(t["PL_NOROW"]), disj(t["PL_MIN"], t["PL_NOROW"]), disj(t["DENSE"], t["PL_NOROW"], t["SHORT"]),
            disj(t["BELOW"], t["PL_MIN"]), disj(t["PL_ROW"], t["PL_NOROW"], t["SHORT2"], t["DENSE"]),
            bq((t["PL_NOROW"], Occur.MUST), (t["PL_MIN"], Occur.SHOULD)),
            bq((t["DENSE"], Occur.MUST), (t["PL_NOROW"], Occur.MUST_NOT), (RangeQuery(0, 10, 300), Occur.FILTER))]


def tie_query(b: Built):
    return disj(b.term["T_TIE"], b.term["D0"], b.term["D1"])


def heavy_query(b: Built):
    return disj(b.term["S_WARM"], b.term["R_RARE"], b.term["D0"], b.term["D1"])
