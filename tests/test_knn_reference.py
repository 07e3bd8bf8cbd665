"""The plain references of the kNN kernel tests (tests/knn_harness.py), checked on the CPU: the bf16 rounding against
torch.bfloat16, the below-midpoint generator, the key layout and the liveDocs bitmap."""
import numpy as np
import torch

import knn_harness as kh


def _torch_bf16(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(torch.bfloat16).to(torch.float32).numpy()


def test_bf16_round_matches_torch():
    rng = np.random.default_rng(3)
    normal = rng.standard_normal(200_000).astype(np.float32) * np.float32(10.0) ** rng.integers(-30, 30, 200_000)
    bits = rng.integers(0, 2**32, 200_000, dtype=np.uint64).astype(np.uint32)
    bits = bits[(bits & 0x7F800000) != 0x7F800000]              # finite values only (Inf / NaN patterns excluded)
    raw = bits.view(np.float32)
    # exact ties (low half 0x8000, even and odd bf16 mantissa) and their fp32 neighbours, subnormals, signed zeros
    hi = rng.integers(0, 0x7F7F, 5_000).astype(np.uint32) << 16
    ties = np.concatenate([hi | 0x8000, hi | 0x7FFF, hi | 0x8001, (hi | 0x8000) | 0x80000000]).view(np.float32)
    special = np.array([0.0, -0.0, 1e-40, -1e-40, 1.17549435e-38, 3.0e38, -3.0e38], np.float32)
    for x in (normal, raw, ties, special):
        got, want = kh.bf16_round(x), _torch_bf16(x)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_below_midpoint_rounds_down_by_almost_half_an_ulp():
    x = kh.below_midpoint(np.random.default_rng(5), (64, 512))
    r = kh.bf16_round(x)
    assert (x > 0).all() and np.array_equal(r, _torch_bf16(x))
    rel = (x.astype(np.float64) - r) / x
    assert (rel > 0).all()                                         # every operand rounds the same way (down)
    assert rel.min() > 2.0**-8 / (1 + 2.0**-6) and rel.max() < 2.0**-8


def test_make_key_orders_score_desc_ordinal_asc():
    scores = np.array([3.5, -1.0, 0.0, 3.5, -7.25, 1e-30, -1e-30, 2.0], np.float32)
    ords = np.array([4, 1, 2, 0, 9, 7, 8, 3], np.int64)
    keys = kh.make_key(scores, ords)
    order = sorted(range(len(keys)), key=lambda i: int(keys[i]), reverse=True)
    want = sorted(range(len(keys)), key=lambda i: (-float(scores[i]), int(ords[i])))
    assert order == want
    assert ((keys & 0xFFFFFFFF) == (~ords.astype(np.uint64) & 0xFFFFFFFF)).all()


def test_live_bits_layout():
    live = np.zeros(70, np.uint8)
    live[[0, 5, 31, 32, 63, 64, 69]] = 1
    w = kh.live_bits(live)
    assert w.dtype == np.uint32 and len(w) == 3
    for d in range(70):
        assert ((int(w[d >> 5]) >> (d & 31)) & 1) == live[d]
