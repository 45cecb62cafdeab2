"""The division-free probability forms of the kernels (ml_prob, half_share in mkp_kernels.cuh) against float32 division.

ml_prob(b) = (b + 0.5) * 2^-8 must give the bits of (b + 0.5) / 256 for every ML byte, and half_share(p) = p * 0.5 the bits
of p / 2 for every probability ReDistribute can halve: one ML probability, or the sum of two (a list's repeated code, or a
code repeated by the next list of the strand). A zero share, 0 / k, is +0, and p + 0 must leave every such p unchanged."""
import numpy as np

F = np.float32


def ml_probs():
    b = np.arange(256, dtype=np.float32)
    return b, (b + F(0.5)) / F(256.0)


def test_ml_prob_matches_division_for_every_byte():
    b, want = ml_probs()
    got = (b + F(0.5)) * F(2.0 ** -8)
    assert got.dtype == np.float32 and want.dtype == np.float32
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_half_share_matches_division_over_every_reachable_probability():
    _, p = ml_probs()
    sums = (p[:, None] + p[None, :]).ravel()
    for v in (p, sums):
        assert v.dtype == np.float32
        assert np.array_equal((v * F(0.5)).view(np.uint32), (v / F(2.0)).view(np.uint32))


def test_zero_share_leaves_probability_unchanged():
    _, p = ml_probs()
    sums = (p[:, None] + p[None, :]).ravel()
    for k in (2.0, 3.0):
        share = F(0.0) / F(k)
        assert share.view(np.uint32) == 0
        for v in (p, sums):
            assert np.array_equal((v + share).view(np.uint32), v.view(np.uint32))
