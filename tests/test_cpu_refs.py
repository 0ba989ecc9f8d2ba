"""CPU: the plain references the GPU tests of the line model and of the segmented sky staging lean
on, pinned against the restatement (oracle/liboracle.so) before a GPU is involved."""
import numpy as np
import pytest

import orcdirac
from util import big_cluster_sky, line_model_ref, relerr, small_problem, split_cluster

needs_oracle = pytest.mark.skipif(not orcdirac.available(), reason="oracle/liboracle.so not built")


@needs_oracle
@pytest.mark.parametrize("nchunk", [None, [1, 3, 2]], ids=["plain", "hybrid"])
def test_line_model_reference_is_the_model_along_the_line(nchunk):
    """V0 + a V1 + a^2 V2 of the numpy line model is the full model at xk + a pk"""
    b = small_problem(N=11, M=3, tilesz=7, seed=81, kmean=1.0, nchunk=nchunk)
    pr = b.pr
    rng = np.random.default_rng(3)
    xk = pr.pp0 + 0.1 * rng.normal(0, 1, pr.pp0.shape)
    pk = 0.05 * rng.normal(0, 1, pr.pp0.shape)
    V0, V1, V2 = line_model_ref(pr, xk, pk)
    orc = orcdirac.Oracle(pr)
    for a in (0.0, 0.7, -2.5):
        assert relerr(V0 + a * V1 + a * a * V2, orc.predict_full(xk + a * pk)) < 1e-14
    assert np.abs(V2).max() > 1e-3 * np.abs(V0).max()   # the quadratic term is not negligible


@needs_oracle
def test_sky_split_identity_on_the_oracle():
    """a cluster's coherencies are the sum of those of its sources split into three clusters of at
    most 96; an empty cluster has zero coherencies"""
    clusters = big_cluster_sky()
    big = clusters[5]                     # 200 sources
    parts = (96, 96, 8)
    rng = np.random.default_rng(1)
    R = 300
    u, v, w = (rng.normal(0, 3e4, R) / 3e8 for _ in range(3))
    whole = orcdirac.OracleSky(clusters).coherencies(u, v, w, 150e6, 2e5).reshape(R, -1, 4)
    split = orcdirac.OracleSky(split_cluster(big, parts)).coherencies(u, v, w, 150e6, 2e5)
    split = split.reshape(R, 3, 4)
    assert relerr(split.sum(axis=1), whole[:, 5]) < 1e-13
    assert not whole[:, 6].any()
    freqs = np.array([146e6, 152e6, 158e6])
    xa = orcdirac.OracleSky([big]).predict_multifreq(u, v, w, freqs, 6e5, 1, np.zeros(8 * R * 3))
    xb = orcdirac.OracleSky(split_cluster(big, parts)).predict_multifreq(u, v, w, freqs, 6e5, 1,
                                                                         np.zeros(8 * R * 3))
    assert relerr(xb, xa) < 1e-13
