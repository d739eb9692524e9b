"""tests/gstep_fixed_point_spec.py is what the CUDA G-step is compared with bit for bit on the GPU; here the specification itself is
pinned on the CPU: against the oracle's restatement of main_responseCalib.cpp:286-304 (the reference's sequential fp64 chain), against
math.fsum (the correctly rounded exact sum) and against itself when the pixels are split into slices the way ranks split them."""
import math

import numpy as np
import pytest

import gstep_fixed_point_spec as fx
from oracle.loader import PortOracle


@pytest.fixture(scope="module")
def port():
    return PortOracle()


def stack(seed, n=31, npix=2000):
    rng = np.random.default_rng(seed)
    data = rng.integers(0, 256, (n, npix), dtype=np.uint8)
    data[:, 3:30] = 255
    data[:, 100:140] = 9
    t = rng.uniform(0.05, 20.0, n)
    E = np.exp(rng.uniform(-10.0, 5.0, npix))
    return data, t, E


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_spec_matches_the_reference_chain_to_rounding_and_the_exact_sum_closely(port, seed):
    data, t, E = stack(seed)
    t[4] = -0.7
    G = fx.gstep(data, t, E)
    G_ref = port.gstep(data, t, E)
    m = np.isfinite(G_ref)
    assert np.array_equal(np.isfinite(G), m)
    assert np.max(np.abs(G[m] - G_ref[m]) / np.abs(G_ref[m])) < 1e-10
    prod = E[None, :] * t[:, None]
    pmax = np.abs(E).max() * np.abs(t).max()
    for b in range(255):
        sel = data == b
        if sel.any():
            exact = math.fsum(prod[sel].tolist()) / int(sel.sum())
            assert abs(G[b] - exact) <= 4e-15 * pmax + 1e-15 * abs(exact)


def test_slices_add_up_to_the_whole_bit_for_bit():
    data, t, E = stack(7, n=19, npix=1500)
    whole = fx.gstep(data, t, E)
    cuts = [0, 384, 385, 1100, 1500]                     # ragged slices, one of a single pixel
    words = np.zeros(4, np.int64)
    for a, b in zip(cuts[:-1], cuts[1:]):
        words = np.maximum(words, fx.scale_words(E[a:b], t))
    limbs, special, counts = np.zeros(768, np.int64), np.zeros(256), np.zeros(256, np.int64)
    for a, b in zip(cuts[:-1], cuts[1:]):
        l, s, c = fx.accumulate(data[:, a:b], t, E[a:b], words)
        limbs += l; special += s; counts += c
    assert np.array_equal(fx.finish(words, limbs, special, counts).view(np.int64), whole.view(np.int64))


@pytest.mark.parametrize("case", ["nan_E", "inf_t", "zero_E", "huge_range", "tiny"])
def test_special_values_follow_the_reference(port, case):
    data, t, E = stack(11, n=13, npix=600)
    if case == "nan_E":
        E[50] = np.nan                                   # poisons exactly the bins pixel 50 has unsaturated samples in
    elif case == "inf_t":
        t[2] = np.inf                                    # the kernels range-check every sample of this pass; the scale stays
    elif case == "zero_E":
        E[:] = 0.0
    elif case == "huge_range":
        E[::7] *= 1e200
        E[1::7] *= 1e-200
    else:
        E *= 1e-250
    with np.errstate(invalid="ignore", over="ignore"):
        G, G_ref = fx.gstep(data, t, E), port.gstep(data, t, E)
    assert np.array_equal(np.isnan(G), np.isnan(G_ref))
    assert np.array_equal(np.isinf(G), np.isinf(G_ref))
    m = np.isfinite(G_ref)
    if case == "inf_t":
        # A non-finite exposure time does not change the scale (it is taken over the finite ones): the bins image 2 does not touch
        # keep the resolution of every other bin.
        direct = np.array([(data == b).any() and not (data[2] == b).any() for b in range(255)] + [False])      # bins with samples, none from image 2
        assert direct.sum() > 20 and np.max(np.abs(G[direct] - G_ref[direct]) / np.abs(G_ref[direct])) <= 1e-10      # (the other finite entries are extrapolations, :300-304)
        return
    # one scale for all bins: a sample is resolved to 2^-48 of the largest product, so that is the error bound of a bin's mean — bins
    # whose products are all 2^48 times smaller than the largest one (only in "huge_range") come out as 0
    fin = np.isfinite(E)
    pmax = np.abs(E[fin]).max() * np.abs(t).max()
    assert np.all(np.abs(G[m] - G_ref[m]) <= 4e-15 * pmax + 1e-10 * np.abs(G_ref[m]))
    if case == "zero_E":
        assert np.all(G[m] == 0.0)


@pytest.mark.parametrize("seed", [4, 5])
def test_vectorised_sums_equal_the_sample_by_sample_sums(seed):
    data, t, E = stack(seed, n=23, npix=700)
    t[3] = -2.5
    E[::13] = -E[::13]
    E[17] = np.nan
    t[5] = np.inf
    words = fx.scale_words(E, t)
    a, b = fx.accumulate(data, t, E, words), fx.accumulate_loop(data, t, E, words)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])
    assert np.array_equal(np.isnan(a[1]), np.isnan(b[1])) and np.array_equal(a[1][~np.isnan(a[1])], b[1][~np.isnan(b[1])])


def test_vectorised_sums_stay_exact_over_many_blocks(monkeypatch):
    """blocks of a few rows: the Python-integer join across bincount blocks, with sums far beyond 2^53 units"""
    data, t, E = stack(6, n=40, npix=900)
    E[:] = np.float64(2.0 ** 20) - 1.0                  # every product near the top of its 2^48-unit range
    words = fx.scale_words(E, t)
    ref = fx.accumulate_loop(data, t, E, words)
    monkeypatch.setattr(fx, "CHUNK", 3 * 900)
    got = fx.accumulate(data, t, E, words)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[2], ref[2])


def extreme(case, seed=13, npix=900):
    """Inputs the C ABI accepts that sit at the edges of the fixed-point scale (and one a `nan` line of times.txt produces)."""
    rng = np.random.default_rng(seed)
    n = 12
    data = rng.integers(0, 255, (n, npix), dtype=np.uint8)
    t = rng.uniform(0.05, 20.0, n)
    E = np.exp(rng.uniform(-10.0, 5.0, npix))
    if case == "tiny_t":                                  # 2^s must exceed 2^1000 for these products to keep 48 bits
        t = rng.uniform(0.5, 2.0, n) * 1e-300
        E = rng.uniform(1.0, 255.0, npix)
    elif case == "tiny_t_large_E":                        # E * 2^s overflows: the scale must go on the product, not on E
        t = rng.uniform(0.5, 2.0, n) * 1e-300
        E = rng.uniform(0.5, 2.0, npix) * 1e8
    elif case == "overflowing_products":                  # max|E| * max|t| and some E * t overflow; the finite bins keep their bits
        E[:300] = rng.uniform(1.0, 2.0, 300) * 1e300
        E[300:] = rng.uniform(0.5, 1.0, npix - 300) * 1e298      # finite products, and bin sums below DBL_MAX
        data[:, :300] = rng.integers(200, 255, (n, 300))
        data[:, 300:] = rng.integers(0, 200, (n, npix - 300))
        t = rng.uniform(0.5, 2.0, n) * 1e8
    elif case in ("nan_t_saturated", "inf_t_saturated"):  # a frame the reference skips entirely must not change anything
        data[3] = 255
        t[3] = np.nan if case == "nan_t_saturated" else np.inf
    elif case in ("nan_t", "inf_t"):                      # an unsaturated frame: its bins are NaN / inf, the others exact
        t[3] = np.nan if case == "nan_t" else -np.inf
        data[3] = rng.integers(0, 20, npix)
    return data, t, E


EXTREME = ["tiny_t", "tiny_t_large_E", "overflowing_products", "nan_t_saturated", "inf_t_saturated", "nan_t", "inf_t"]


def assert_matches_reference(G, G_ref, what, tol=1e-10):
    assert np.array_equal(np.isnan(G), np.isnan(G_ref)), f"{what}: NaN masks differ"
    assert np.array_equal(np.isposinf(G), np.isposinf(G_ref)) and np.array_equal(np.isneginf(G), np.isneginf(G_ref)), f"{what}: inf masks differ"
    m = np.isfinite(G_ref)
    rel = np.abs(G[m] - G_ref[m]) / np.abs(G_ref[m])
    assert m.any() and np.max(rel) <= tol, f"{what}: {np.max(rel):.3g} relative from the reference"


@pytest.mark.parametrize("case", EXTREME)
def test_extreme_values_against_the_reference(port, case):
    data, t, E = extreme(case)
    with np.errstate(invalid="ignore", over="ignore"):
        G, G_ref = fx.gstep(data, t, E), port.gstep(data, t, E)
    assert_matches_reference(G, G_ref, case)
    if case in ("nan_t", "inf_t"):
        assert not np.all(np.isfinite(G_ref[:20]))
