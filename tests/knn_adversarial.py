"""Corpora on which a bf16 candidate stage provably ranks wrong, for the tests of the kNN rank-safety certificate.

One adversarial query has every component equal to one value just below a bf16 rounding midpoint. Its k true
neighbours are permutations of one vector whose components also sit just below midpoints: both operands round down, so
their bf16 scores read about 2^-7 low. More than k' decoys are exact in bf16 (only the query's rounding, about 2^-8,
touches their scores) and their true scores lie in between: above the neighbours in bf16, below them exactly. The bf16
top-k' therefore holds decoys only, and the page re-scored from it is wrong: only a sound certificate saves the query.
Gaussian fillers and Gaussian control queries (which a correct certificate accepts) complete the corpus.

Everything here is numpy on the CPU; tests/test_knn_adversarial_reference.py proves these facts for every builder."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import knn_stage_b as kh

DIMS = 64
WARM, CHUNK1 = 32768, 65536   # kKnnWarmChunk and the first fused chunk of knn_search_host


@dataclass
class Adversarial:
    sim: int
    k: int
    kprime: int
    corpus: np.ndarray       # float32 [n][DIMS]
    queries: np.ndarray      # float32 [nq][DIMS]: n_adv adversarial queries first, then Gaussian controls
    n_adv: int
    neighbours: np.ndarray   # ordinals of the k true neighbours of every adversarial query
    decoys: np.ndarray       # ordinals of the decoys


def kprime_of(k: int) -> int:
    """Candidates per query of the tensor-core stage (knn_search_host)."""
    return min(max(128, 4 * k), 4096 - 256)


def approx_bf16(Q, D, sim: int) -> np.ndarray:
    """float64 candidate scores as the bf16 stage sees them: rounded operands, the true |d|^2 of the index."""
    n2 = (np.asarray(D, np.float64) ** 2).sum(axis=1).astype(np.float32)
    return kh.approx_reference(kh.bf16_round(Q), kh.bf16_round(D), sim, norm2=n2)


def _decoys(rng, q, base, sim, want, a_nb_bf16, a_nb_true, unit):
    """bf16-exact vectors near permutations of `base` whose candidate score beats the neighbours' in bf16 and loses to
    it exactly, each by at least 2 % of the certificate's bound (unit). Kept by rejection."""
    out = []
    for _ in range(40):
        m = 8 * want
        p = np.stack([rng.permutation(base) for _ in range(m)]).astype(np.float64)
        scale = rng.uniform(0.985, 1.003, (m, 1))
        spread = rng.uniform(0.0, 0.06, (m, 1))       # widening the components about their mean lowers the cosine
        d = kh.bf16_round(((p + spread * (p - p.mean(axis=1, keepdims=True))) * scale).astype(np.float32))
        ok = (approx_bf16(q[None, :], d, sim)[0] > a_nb_bf16 + 0.02 * unit) & \
             (kh.approx_reference(q[None, :], d, sim)[0] < a_nb_true - 0.02 * unit)
        out.extend(d[ok])
        if len(out) >= want:
            return np.stack(out[:want])
    raise AssertionError(f"only {len(out)} of {want} decoys found")


def build(sim: int, k: int = 10, seed: int = 0, n_fill: int = 3000, n_ctrl: int = 4, n_adv: int = 3, fused: bool = False,
          qscale: float = 2.0) -> Adversarial:
    """sim: a float similarity. fused = False: a corpus inside the warm chunk (knn_select_kernel alone builds the
    lists). fused = True: fillers fill the warm chunk, the decoys lie in the first fused chunk and the neighbours in the
    second, so it is the fused epilogue's threshold that drops them."""
    rng = np.random.default_rng(seed + 1000 * sim + k)
    kp = kprime_of(k)
    base = kh.below_midpoint(rng, DIMS, exp_lo=-1, exp_hi=0)
    # the adversarial queries: one value in every component, 1, 2, ... fp32 ulps below the midpoint 1 + 2^-8 (so the
    # queries differ, yet one decoy set serves them all)
    qv = (np.uint32(0x3F808000) - np.arange(1, n_adv + 1, dtype=np.uint32)).view(np.float32)
    adv_q = (np.ones((n_adv, DIMS), np.float32) * qv[:, None])
    adv_q = (adv_q * np.float32(qscale)).astype(np.float32)    # a power of two keeps the components below midpoints
    nb = np.stack([rng.permutation(base) for _ in range(k)]).astype(np.float32)
    dmax = float(np.linalg.norm(nb[0].astype(np.float64))) * 1.003 * 1.06
    qn = np.linalg.norm(adv_q.astype(np.float64), axis=1)
    a_bf = approx_bf16(adv_q, nb, sim).max(axis=1)
    a_tr = kh.approx_reference(adv_q, nb, sim).min(axis=1)
    units = np.array([kh.approx_unit(sim, qn[i], dmax, 2.0**-7) for i in range(n_adv)])
    decoys = _decoys(rng, adv_q[0], base, sim, kp + 24, a_bf[0], a_tr[0], units[0])
    fill = rng.standard_normal((n_fill, DIMS)).astype(np.float32)
    fill *= np.float32(0.9 * np.linalg.norm(nb[0]) / np.sqrt(DIMS))
    ctrl = rng.standard_normal((n_ctrl, DIMS)).astype(np.float32)
    if fused:
        warm = rng.standard_normal((WARM, DIMS)).astype(np.float32) * np.float32(0.9 * np.linalg.norm(nb[0]) / np.sqrt(DIMS))
        mid = rng.standard_normal((CHUNK1 - len(decoys), DIMS)).astype(np.float32) * np.float32(0.9 * np.linalg.norm(nb[0]) / np.sqrt(DIMS))
        corpus = np.concatenate([warm, decoys, mid, fill[:500], nb, fill[500:]])
        dec0, nb0 = WARM, WARM + CHUNK1 + 500
    else:
        corpus = np.concatenate([nb, fill[:700], decoys, fill[700:]])
        nb0, dec0 = 0, k + 700
    return Adversarial(sim, k, kp, np.ascontiguousarray(corpus, np.float32), np.concatenate([adv_q, ctrl]).astype(np.float32),
                       n_adv, np.arange(nb0, nb0 + k), np.arange(dec0, dec0 + len(decoys)))


def brute_force(adv: Adversarial, boosts=None):
    """fp64 brute-force pages of every query: (docs [nq][k], scores [nq][k]) by (score desc, ordinal asc)."""
    s = kh.exact_scores(adv.queries, adv.corpus, adv.sim, boosts)
    pages = [kh.page_reference(s[q], adv.k) for q in range(len(s))]
    return np.stack([p[0] for p in pages]), np.stack([p[1] for p in pages])
