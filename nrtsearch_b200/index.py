"""Host-side shard description (what the adaptor extracts from Lucene LeafReaders at
ShardSearcherFactory.newSearcher, reference src/main/java/com/yelp/nrtsearch/server/index/ShardState.java:506-526)
and the deterministic synthetic corpora of SURVEY.md Appendix B."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

from . import _native

SEED_CORPUS = 0x5EED0001
SEED_QUERIES = 0x5EED0002
SEED_VECTORS = 0x5EED0003
SEED_VQUERIES = 0x5EED0004
SEED_PRICE = 0x5EED0005
SEED_RANGE = 0x5EED0006

SIM_L2, SIM_DOT, SIM_COSINE, SIM_MIP = 0, 1, 2, 3


@dataclass
class TextField:
    """Per text field: norms column + INDEX-WIDE collection statistics (BM25 needs global stats)."""
    norms: Optional[np.ndarray]  # uint8[n_docs] SmallFloat.intToByte4(length); None = omitNorms
    doc_count: int
    sum_total_term_freq: int
    k1: float = 1.2
    b: float = 0.75


@dataclass
class KeywordColumn:
    """String doc values of one keyword field in one leaf (SortedDocValues / SortedSetDocValues): the leaf's term
    dictionary, strictly ascending in byte order, and each doc's ordinals into it. SORTED (offsets None): ords is
    int32[n_docs], -1 for a doc without a value. SORTED_SET: offsets is int64[n_docs+1] and ords the flattened ordinals,
    strictly ascending within a doc (the set Lucene keeps: each term of a doc once)."""
    terms: List[bytes]
    ords: np.ndarray
    offsets: Optional[np.ndarray] = None

    @staticmethod
    def from_values(values: Sequence, multi_valued: bool) -> "KeywordColumn":
        """The column of per-doc values as an adaptor reads them from documents: SORTED, a str / bytes or None per doc;
        SORTED_SET, an iterable of them per doc (repeats collapse, as in SortedSetDocValues)."""
        enc = [(None if v is None else _utf8(v)) if not multi_valued else sorted({_utf8(x) for x in v}) for v in values]
        terms = sorted({t for v in enc for t in ([v] if not multi_valued else v) if t is not None})
        ord_of = {t: i for i, t in enumerate(terms)}
        if not multi_valued:
            return KeywordColumn(terms, np.array([-1 if v is None else ord_of[v] for v in enc], np.int32))
        off = np.zeros(len(enc) + 1, np.int64)
        np.cumsum([len(v) for v in enc], out=off[1:])
        return KeywordColumn(terms, np.array([ord_of[t] for v in enc for t in v], np.int32), off)

    @property
    def multi_valued(self) -> bool:
        return self.offsets is not None

    def doc_ords(self, doc: int) -> np.ndarray:
        if self.offsets is None:
            o = int(self.ords[doc])
            return np.zeros(0, np.int32) if o < 0 else np.array([o], np.int32)
        return self.ords[int(self.offsets[doc]):int(self.offsets[doc + 1])]

    def doc_range(self, lo: int, hi: int) -> "KeywordColumn":
        """The column of docs [lo, hi) as a segment of them holds it: its own dictionary, only the terms present there,
        ordinals renumbered."""
        if self.offsets is None:
            sub = self.ords[lo:hi]
        else:
            sub = self.ords[int(self.offsets[lo]):int(self.offsets[hi])]
        present = np.unique(sub[sub >= 0])
        remap = np.full(len(self.terms) + 1, -1, np.int32)
        remap[present] = np.arange(len(present), dtype=np.int32)
        ords = np.ascontiguousarray(remap[sub], np.int32)
        terms = [self.terms[int(t)] for t in present]
        if self.offsets is None:
            return KeywordColumn(terms, ords)
        return KeywordColumn(terms, ords, np.ascontiguousarray(self.offsets[lo:hi + 1] - self.offsets[lo]))


def _utf8(v) -> bytes:
    return v.encode("utf-8") if isinstance(v, str) else bytes(v)


@dataclass
class HostShard:
    n_docs: int
    doc_base: int
    term_off: np.ndarray      # int64[n_terms+1]
    post_docs: np.ndarray     # int32[P], shard-local ids
    post_freqs: np.ndarray    # int32[P]
    fields: List[TextField]
    term_field: Optional[np.ndarray] = None   # int32[n_terms]
    term_df: Optional[np.ndarray] = None      # int64[n_terms] index-wide docFreq
    columns: List[np.ndarray] = field(default_factory=list)        # int64[n_docs] each
    column_has: List[Optional[np.ndarray]] = field(default_factory=list)
    # multi-valued columns (SORTED_NUMERIC): column_offsets[i] = int64[n_docs+1], columns[i] = the flattened values
    # (ascending within a doc); None / missing entry = single-valued column
    column_offsets: List[Optional[np.ndarray]] = field(default_factory=list)
    live_docs: Optional[np.ndarray] = None    # uint8[n_docs]
    vectors: Optional[np.ndarray] = None      # float32[n_vec, dims]
    vec_similarity: int = SIM_COSINE
    vec_docs: Optional[np.ndarray] = None     # int32[n_vec] ord -> doc
    # term positions (PostingsEnum.POSITIONS): posting after posting, the post_freqs[p] positions of posting p, ascending;
    # None = indexed without positions (PhraseQuery is refused)
    post_positions: Optional[np.ndarray] = None
    # keyword columns (string doc values, nrtgpu_index_add_keyword_columns); keyword column k is TermsCollector(k, ...,
    # field_type="keyword")
    keyword_columns: List[KeywordColumn] = field(default_factory=list)
    # block joins (NestedQuery): the term every parent doc holds (_nested_path:_root); each parent follows its child docs.
    # None = an index without nested documents (NestedQuery is refused)
    parent_term: Optional[int] = None

    @property
    def n_terms(self) -> int:
        return len(self.term_off) - 1

    def _mv(self, i: int) -> Optional[np.ndarray]:
        return self.column_offsets[i] if i < len(self.column_offsets) else None

    def df(self, term: int) -> int:
        return int(self.term_off[term + 1] - self.term_off[term])

    def doc_range(self, lo: int, hi: int, doc_base: Optional[int] = None) -> "HostShard":
        """Contiguous doc-range sub-shard [lo, hi) keeping the index-wide statistics (SURVEY.md 8e)."""
        nt = self.n_terms
        starts = np.empty(nt, dtype=np.int64)
        ends = np.empty(nt, dtype=np.int64)
        # postings are doc-sorted per term: find the sub-range of every list
        for t in range(nt):
            a, b = int(self.term_off[t]), int(self.term_off[t + 1])
            seg = self.post_docs[a:b]
            starts[t] = a + np.searchsorted(seg, lo, side="left")
            ends[t] = a + np.searchsorted(seg, hi, side="left")
        lens = ends - starts
        off = np.zeros(nt + 1, dtype=np.int64)
        np.cumsum(lens, out=off[1:])
        idx = np.concatenate([np.arange(s, e, dtype=np.int64) for s, e in zip(starts, ends)]) if nt else np.zeros(0, np.int64)
        global_df = self.term_df if self.term_df is not None else np.diff(self.term_off)
        sub_pos = None
        if self.post_positions is not None:   # the positions of the kept postings, in their order
            pstart = np.zeros(len(self.post_freqs) + 1, np.int64)
            np.cumsum(self.post_freqs, out=pstart[1:])
            f = self.post_freqs[idx].astype(np.int64)
            first = np.repeat(pstart[idx] - (np.cumsum(f) - f), f)
            sub_pos = np.ascontiguousarray(self.post_positions[first + np.arange(int(f.sum()), dtype=np.int64)], np.int32)
        sub_vec = sub_vdocs = None
        if self.vectors is not None:
            vd = self.vec_docs if self.vec_docs is not None else np.arange(len(self.vectors), dtype=np.int32)
            m = (vd >= lo) & (vd < hi)
            sub_vec = np.ascontiguousarray(self.vectors[m])
            sub_vdocs = (vd[m] - lo).astype(np.int32)
        return HostShard(
            n_docs=hi - lo, doc_base=(self.doc_base + lo) if doc_base is None else doc_base, term_off=off,
            post_docs=(self.post_docs[idx] - lo).astype(np.int32), post_freqs=np.ascontiguousarray(self.post_freqs[idx]),
            fields=[TextField(None if f.norms is None else np.ascontiguousarray(f.norms[lo:hi]), f.doc_count,
                              f.sum_total_term_freq, f.k1, f.b) for f in self.fields],
            term_field=self.term_field, term_df=np.ascontiguousarray(global_df.astype(np.int64)),
            columns=[np.ascontiguousarray(c[lo:hi]) if self._mv(i) is None else
                     np.ascontiguousarray(c[int(self._mv(i)[lo]):int(self._mv(i)[hi])]) for i, c in enumerate(self.columns)],
            column_offsets=[None if self._mv(i) is None else np.ascontiguousarray(self._mv(i)[lo:hi + 1] - self._mv(i)[lo])
                            for i in range(len(self.columns))],
            column_has=[None if h is None else np.ascontiguousarray(h[lo:hi]) for h in self.column_has],
            live_docs=None if self.live_docs is None else np.ascontiguousarray(self.live_docs[lo:hi]),
            vectors=sub_vec, vec_similarity=self.vec_similarity, vec_docs=sub_vdocs, post_positions=sub_pos,
            keyword_columns=[k.doc_range(lo, hi) for k in self.keyword_columns], parent_term=self.parent_term)


def _ptr(a: Optional[np.ndarray], typ):
    if a is None:
        return C.cast(None, typ)
    return a.ctypes.data_as(typ)


class PinnedDesc:
    """Keeps the numpy arrays alive while a C shard descriptor points at them."""

    def __init__(self, sh: HostShard):
        N = _native
        self.keep = []

        def arr(a, dt):
            if a is None:
                return None
            b = np.ascontiguousarray(a, dtype=dt)
            self.keep.append(b)
            return b

        d = N.ShardDesc()
        d.n_docs, d.doc_base, d.n_terms = sh.n_docs, sh.doc_base, sh.n_terms
        d.term_off = _ptr(arr(sh.term_off, np.int64), N.i64p)
        d.post_docs = _ptr(arr(sh.post_docs, np.int32), N.i32p)
        d.post_freqs = _ptr(arr(sh.post_freqs, np.int32), N.i32p)
        d.term_field = _ptr(arr(sh.term_field, np.int32), N.i32p)
        d.term_df = _ptr(arr(sh.term_df, np.int64), N.i64p)
        nf = len(sh.fields)
        d.n_fields = nf
        norms = (N.u8p * max(nf, 1))()
        for i, f in enumerate(sh.fields):
            norms[i] = _ptr(arr(f.norms, np.uint8), N.u8p)
        self.keep.append(norms)
        d.norms = C.cast(norms, C.POINTER(N.u8p))
        d.field_doc_count = _ptr(arr(np.array([f.doc_count for f in sh.fields], np.int64), np.int64), N.i64p)
        d.field_sum_ttf = _ptr(arr(np.array([f.sum_total_term_freq for f in sh.fields], np.int64), np.int64), N.i64p)
        d.field_k1 = _ptr(arr(np.array([f.k1 for f in sh.fields], np.float32), np.float32), N.f32p)
        d.field_b = _ptr(arr(np.array([f.b for f in sh.fields], np.float32), np.float32), N.f32p)
        nc = len(sh.columns)
        d.n_columns = nc
        cols = (N.i64p * max(nc, 1))()
        has = (N.u8p * max(nc, 1))()
        for i, c in enumerate(sh.columns):
            cols[i] = _ptr(arr(c, np.int64), N.i64p)
            h = sh.column_has[i] if i < len(sh.column_has) else None
            has[i] = _ptr(arr(h, np.uint8), N.u8p)
        offs = (N.i64p * max(nc, 1))()
        for i in range(nc):
            offs[i] = _ptr(arr(sh._mv(i), np.int64), N.i64p)
        self.keep += [cols, has, offs]
        d.columns = C.cast(cols, C.POINTER(N.i64p))
        d.column_has = C.cast(has, C.POINTER(N.u8p))
        d.column_offsets = C.cast(offs, C.POINTER(N.i64p))
        d.live_docs = _ptr(arr(sh.live_docs, np.uint8), N.u8p)
        if sh.vectors is not None and len(sh.vectors):
            byte_field = np.asarray(sh.vectors).dtype == np.int8   # ByteVectorFieldDef
            v = arr(sh.vectors, np.int8 if byte_field else np.float32)
            d.vec_dims, d.vec_similarity, d.vec_count = v.shape[1], sh.vec_similarity, v.shape[0]
            d.vectors = v.ctypes.data
            d.vec_element_type = 1 if byte_field else 0
            d.vec_docs = _ptr(arr(sh.vec_docs, np.int32), N.i32p)
        self.desc = d
        # keyword columns (nrtgpu_index_add_keyword_columns, after the build)
        self.keyword = (N.KeywordColumn * max(len(sh.keyword_columns), 1))()
        for i, k in enumerate(sh.keyword_columns):
            toff = np.zeros(len(k.terms) + 1, np.int64)
            np.cumsum([len(t) for t in k.terms], out=toff[1:])
            tb = arr(np.frombuffer(b"".join(k.terms) or b"\0", np.uint8), np.uint8)
            self.keyword[i] = N.KeywordColumn(len(k.terms), 1 if k.multi_valued else 0, tb.ctypes.data, arr(toff, np.int64).ctypes.data,
                                              arr(k.ords, np.int32).ctypes.data,
                                              None if k.offsets is None else arr(k.offsets, np.int64).ctypes.data)
        self.n_keyword = len(sh.keyword_columns)


# ---------------------------------------------------------------- synthetic inputs (Appendix B)

def synth_text_shard(n_docs: int, vocab: int, seed: int = SEED_CORPUS, min_len: int = 8,
                     poisson_mean: float = 56.0, zipf_s: float = 1.0, doc_begin: int = 0) -> HostShard:
    """Zipf(s) token stream, doc length = min_len + Poisson(mean); single text field with norms.
    The shard holds global docs [doc_begin, doc_begin+n_docs) of the (unbounded) synthetic corpus with
    doc_base = doc_begin; statistics are SHARD-LOCAL until the caller installs index-wide ones."""
    lib = _native.synth_lib()
    df = np.zeros(vocab, dtype=np.int64)
    norms = np.zeros(n_docs, dtype=np.uint8)
    ttf, npost = C.c_int64(0), C.c_int64(0)
    h = lib.nrtsynth_corpus_begin(n_docs, doc_begin, vocab, seed, min_len, poisson_mean, zipf_s, df.ctypes.data,
                                  norms.ctypes.data, C.byref(ttf), C.byref(npost))
    try:
        term_off = np.zeros(vocab + 1, dtype=np.int64)
        docs = np.empty(npost.value, dtype=np.int32)
        freqs = np.empty(npost.value, dtype=np.int32)
        lib.nrtsynth_corpus_fill(h, term_off.ctypes.data, docs.ctypes.data, freqs.ctypes.data)
    finally:
        lib.nrtsynth_corpus_end(h)
    return HostShard(n_docs=n_docs, doc_base=doc_begin, term_off=term_off, post_docs=docs, post_freqs=freqs,
                     fields=[TextField(norms, n_docs, int(ttf.value))])


def synth_int_column(n_docs: int, value_range: int = 1_000_000, seed: int = SEED_PRICE, doc_begin: int = 0) -> np.ndarray:
    out = np.empty(n_docs, dtype=np.int32)
    _native.synth_lib().nrtsynth_int_column(n_docs, doc_begin, seed, value_range, out.ctypes.data)
    return out.astype(np.int64)


def synth_query_terms(nq: int, terms_per_query: int, vocab: int, seed: int = SEED_QUERIES,
                      log10_lo: float = 1.0, log10_hi: float = 4.0) -> np.ndarray:
    """Distinct term ranks per query, log-uniform in [10^lo, 10^hi) (clamped to the vocabulary)."""
    out = np.empty((nq, terms_per_query), dtype=np.int32)
    _native.synth_lib().nrtsynth_queries(nq, terms_per_query, seed, log10_lo, log10_hi, vocab, out.ctypes.data)
    return out


def synth_uniform(n: int, seed: int) -> np.ndarray:
    out = np.empty(n, dtype=np.float64)
    _native.synth_lib().nrtsynth_uniform(n, seed, out.ctypes.data)
    return out


def synth_vectors(n: int, dims: int, seed: int = SEED_VECTORS, row_begin: int = 0) -> np.ndarray:
    assert (row_begin * dims) % 2 == 0
    out = np.empty((n, dims), dtype=np.float32)
    _native.synth_lib().nrtsynth_normal_f32(n * dims, row_begin * dims, seed, out.ctypes.data)
    return out
