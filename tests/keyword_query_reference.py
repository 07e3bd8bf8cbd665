"""Reference for keyword range and prefix queries and keyword value sets (TermRangeQuery, PrefixQuery and
SetQueryFilter over the TEXTTERMS of an atom field), the checker of NRTGPU_KEYWORD_RANGE and
NRTGPU_AGG_FILTER_KEYWORD_SET. TEST INFRASTRUCTURE ONLY.

A plain restatement of the rules over each doc's terms as Python bytes, independent of the library's codes:
  - a range matches a term t when lower <= t (lower < t when exclusive; no lower bound: always) and t <= upper (t < upper
    when exclusive; no upper bound: always), bytes compared as BytesRef.compareTo does (Python's bytes order);
  - a prefix p matches a term t when t starts with p;
  - a value set matches a term t when t is one of its values;
  - a doc matches when one of its terms does (one term for a SORTED column, any of them for a SORTED_SET one); a doc
    without a value never matches."""
from typing import Callable, List, Optional

import numpy as np


def range_pred(lower: Optional[bytes], upper: Optional[bytes], include_lower: bool = True,
               include_upper: bool = True) -> Callable[[bytes], bool]:
    def pred(t: bytes) -> bool:
        if lower is not None and (t < lower or (t == lower and not include_lower)):
            return False
        if upper is not None and (t > upper or (t == upper and not include_upper)):
            return False
        return True
    return pred


def prefix_pred(prefix: bytes) -> Callable[[bytes], bool]:
    return lambda t: t.startswith(prefix)


def set_pred(values) -> Callable[[bytes], bool]:
    s = {bytes(v) for v in values}
    return lambda t: t in s


def doc_terms(col) -> List[List[bytes]]:
    """each doc's terms of keyword column col (index.KeywordColumn) as bytes"""
    if not col.multi_valued:
        return [[] if o < 0 else [bytes(col.terms[int(o)])] for o in col.ords]
    return [[bytes(col.terms[int(o)]) for o in col.ords[col.offsets[d]:col.offsets[d + 1]]] for d in range(len(col.offsets) - 1)]


def match_mask(col, pred: Callable[[bytes], bool]) -> np.ndarray:
    """bool [n_docs]: the docs one of whose terms pred matches"""
    hit = {bytes(t): pred(bytes(t)) for t in col.terms}
    return np.array([any(hit[t] for t in ts) for ts in doc_terms(col)], bool)


def matching_terms(terms, pred: Callable[[bytes], bool]) -> List[bytes]:
    return [bytes(t) for t in terms if pred(bytes(t))]
