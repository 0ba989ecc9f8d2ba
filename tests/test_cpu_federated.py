"""CPU tier of the federated stochastic calibration's host steps (sagecal-mpi -N -M -w -A, the stochastic
slave): dirac_b200_consensus_prod_inverse_fed against the reference's find_prod_inverse_full_fed, and
dirac_b200_federated_bands_update against the slave's lines (sagecal_stochastic_slave.cpp:731-852)
restated in numpy around the reference's own update_global_z_multi.

The tests call the reference first and the product library afterwards, so that the reference's answers
can be recorded (tests/golden/ref/test_cpu_federated)."""
import ctypes as C

import numpy as np
import pytest

from test_cpu_stochastic_consensus import MT, N, ref_basis, ref_prod_inverse, restated_update

RES_RATIO = 1.5       # sagecal_stochastic_slave.cpp res_ratio
CLM_DBL_MAX = 1e12    # Dirac_common.h
vp = C.c_void_p


@pytest.fixture(scope="module")
def capi():
    from sagecal_b200 import lib
    return lib.load()


def _p(a):
    return a.ctypes.data_as(vp)


def ref_prod_inverse_fed(ref, B, rhok, alphak):
    nsolbw, Npoly = B.shape
    Bi = np.zeros((rhok.shape[1], Npoly, Npoly))
    ref.lib.find_prod_inverse_full_fed.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int]
    ref.lib.find_prod_inverse_full_fed(_p(B), _p(Bi), Npoly, nsolbw, rhok.shape[1], _p(rhok),
                                       _p(alphak), 2)
    return Bi


@pytest.mark.parametrize("Npoly", [1, 2, 3])
@pytest.mark.parametrize("nsolbw", [2, 4])
def test_prod_inverse_fed_matches_the_reference(ref, capi, Npoly, nsolbw):
    """(sum_f rho B_f B_f^T + alpha I)^-1, with fewer bands than terms (singular sums) included"""
    rng = np.random.default_rng(10 * Npoly + nsolbw)
    ffreq = np.linspace(140e6, 160e6, nsolbw)
    rhok = np.ascontiguousarray(rng.uniform(2.0, 8.0, (nsolbw, MT)))
    alphak = rng.uniform(0.5, 3.0, MT)
    B = ref_basis(ref, Npoly, ffreq, 150e6, 2)
    want = ref_prod_inverse_fed(ref, B, rhok, alphak)
    got = capi.consensus_prod_inverse_fed(B, rhok, alphak)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def restated_fed_update(ref, admm, r00, r01, J, B, Bi, rhok, alphak, Zavg, X, Y):
    """sagecal_stochastic_slave.cpp:731-852 in numpy around the reference's update_global_z_multi, one
    MS; returns (res_0, res_1, fband, Y, Z)"""
    nsolbw, Npoly = B.shape
    n8 = 8 * N
    res_0 = np.sum(r00) / nsolbw                     # reset for every minibatch (:731, 757-758)
    res_1 = np.sum(r01) / nsolbw
    resband = np.where((r00 > 0.0) & (r01 > 0.0), r01, CLM_DBL_MAX)
    fband = np.array([1 if resband[b] > RES_RATIO * res_1 else 0 for b in range(nsolbw)], np.int32)
    Y = Y.copy()
    rho_i = np.repeat(rhok, n8, axis=1)
    for b in range(nsolbw):
        if not fband[b]:
            Y[b] += rho_i[b] * J[b]
    if not fband[0]:                                  # :783-790
        z = B[0][:, None] * Y[0][None, :]
    else:
        z = np.zeros((Npoly, Y.shape[1]))
    for b in range(1, nsolbw):
        if not fband[b]:
            z += B[b][:, None] * Y[b][None, :]
    z = z.reshape(Npoly, MT, n8)
    if admm > 0:                                      # :805-826, z [Npoly][Mt] vs Zavg, X [Mt][Npoly]
        for ci in range(MT):
            for p in range(Npoly):
                z[p, ci] += alphak[ci] * Zavg[ci, p]
                z[p, ci] += -1.0 * X[ci, p]
    z = np.ascontiguousarray(z)
    Z = np.zeros((MT, Npoly, n8))
    ref.lib.update_global_z_multi.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int]
    ref.lib.update_global_z_multi(_p(Z), N, MT, Npoly, _p(z), _p(np.ascontiguousarray(Bi)), 2)
    for b in range(nsolbw):
        if not fband[b]:
            bz = np.einsum("p,kpi->ki", B[b], Z).reshape(-1)
            Y[b] -= rho_i[b] * bz
    return res_0, res_1, fband, Y, Z


def _close(got, want, tol=1e-14):
    return np.max(np.abs(got - want)) <= tol * np.max(np.abs(want))


CASES = ["all-good", "middle-flagged", "band0-flagged", "nonpositive-cost", "nan-band"]


@pytest.mark.parametrize("admm", [0, 1])
@pytest.mark.parametrize("Npoly", [1, 3])
@pytest.mark.parametrize("case", CASES)
def test_federated_bands_update_matches_the_slave(ref, capi, case, Npoly, admm):
    nsolbw = 3
    rng = np.random.default_rng(300 + 10 * Npoly + CASES.index(case) + 100 * admm)
    m = 8 * N * MT
    ffreq = np.array([143e6, 151e6, 158e6])
    rhok = np.ascontiguousarray(rng.uniform(2.0, 8.0, (nsolbw, MT)))
    alphak = rng.uniform(0.5, 2.0, MT)
    J = rng.normal(0, 1, (nsolbw, m))
    Y = rng.normal(0, 0.5, (nsolbw, m))
    Zavg = rng.normal(0, 1, (MT, Npoly, 8 * N))
    X = rng.normal(0, 0.3, (MT, Npoly, 8 * N))
    r00 = rng.uniform(1.0, 2.0, nsolbw)
    r01 = rng.uniform(0.5, 0.9, nsolbw)
    if case == "middle-flagged":
        r01[1] = 10.0
    elif case == "band0-flagged":
        r01[0] = 10.0
    elif case == "nonpositive-cost":
        r00[2] = 0.0                                  # counts as CLM_DBL_MAX: flagged
    elif case == "nan-band":
        r00[2] = r01[2] = np.nan                      # a band without channels
    B = ref_basis(ref, Npoly, ffreq, 150e6, 2)
    Bi = ref_prod_inverse_fed(ref, B, rhok, alphak)
    w0, w1, wf, wY, wZ = restated_fed_update(ref, admm, r00, r01, J, B, Bi, rhok, alphak, Zavg, X, Y)
    want_flags = {"all-good": [0, 0, 0], "middle-flagged": [0, 1, 0], "band0-flagged": [1, 0, 0],
                  "nonpositive-cost": [0, 0, 1], "nan-band": [0, 0, 0]}[case]
    assert list(wf) == want_flags

    Yg = Y.copy()
    Zg = np.full((MT, Npoly, 8 * N), 123.0)
    rv, g0, g1, gf = capi.federated_bands_update(N, admm, r00, r01, J, B, Bi, rhok, alphak, Zavg, X,
                                                 Yg, Zg)
    assert rv == 0
    assert list(gf) == list(wf)
    for g, w in ((g0, w0), (g1, w1)):
        assert (np.isnan(g) and np.isnan(w)) or abs(g - w) <= 1e-14 * abs(w)
    assert _close(Zg, wZ)
    assert _close(Yg, wY)
    if case == "band0-flagged":
        assert np.array_equal(Yg[0], Y[0])            # neither updated nor summed into z


def test_federated_step_differs_from_the_in_process_step(ref, capi):
    """the same inputs through dirac_b200_consensus_bands_update: a flagged band 0 is summed there and
    not here, and res_0 / res_1 mix with the previous values there and are reset here"""
    nsolbw, Npoly = 3, 2
    rng = np.random.default_rng(77)
    m = 8 * N * MT
    rhok = np.ascontiguousarray(rng.uniform(2.0, 8.0, (nsolbw, MT)))
    J = rng.normal(0, 1, (nsolbw, m))
    Y = rng.normal(0, 0.5, (nsolbw, m))
    r00 = rng.uniform(1.0, 2.0, nsolbw)
    r01 = np.array([10.0, 0.6, 0.7])                  # band 0 flagged
    B = ref_basis(ref, Npoly, np.array([143e6, 151e6, 158e6]), 150e6, 2)
    Bi = ref_prod_inverse(ref, B, rhok)
    _, _, _, wY, wZ = restated_update(ref, r00, r01, J, B, Bi, rhok, 1.3, 0.7, Y)
    Zc = np.zeros((MT, Npoly, 8 * N))
    Yc = Y.copy()
    _, c0, c1, cf = capi.consensus_bands_update(N, r00, r01, J, B, Bi, rhok, 1.3, 0.7, Yc, Zc)
    Zf = np.zeros((MT, Npoly, 8 * N))
    Yf = Y.copy()
    zero = np.zeros((MT, Npoly, 8 * N))
    _, f0, f1, ff = capi.federated_bands_update(N, 0, r00, r01, J, B, Bi, rhok, np.ones(MT), zero,
                                                zero, Yf, Zf)
    assert list(cf) == list(ff) == [1, 0, 0]
    assert _close(Zc, wZ) and not np.allclose(Zc, Zf)
    assert abs(f1 - np.mean(r01)) <= 1e-15 * f1 and abs(c1 - (0.7 + np.sum(r01)) / 3) <= 1e-15 * c1
    assert abs(f0 - np.mean(r00)) <= 1e-15 * f0 and abs(c0 - (1.3 + np.sum(r00)) / 3) <= 1e-15 * c0


def test_federated_bands_update_refuses_bad_sizes(capi):
    """no bands, no polynomial terms or a negative ADMM iteration: -1, nothing touched"""
    Y = np.ones((1, 8 * N * MT))
    Z = np.ones((MT, 1, 8 * N))
    zero = np.zeros((MT, 1, 8 * N))
    for B, admm in ((np.ones((0, 1)), 0), (np.ones((1, 0)), 0), (np.ones((1, 1)), -1)):
        rv, r0, r1, _ = capi.federated_bands_update(N, admm, np.ones(1), np.ones(1), Y, B,
                                                    np.ones((MT, 1, 1)), np.ones((1, MT)),
                                                    np.ones(MT), zero, zero, Y, Z)
        assert rv == -1 and (r0, r1) == (0.0, 0.0)
    assert (Y == 1).all() and (Z == 1).all()


def test_federated_term_goes_to_every_chunk_of_a_hybrid_sky(capi):
    """Mt = 4 chunks of M = 3 clusters (one cluster with two hybrid chunks): the term
    alpha_k Zavg[k][p] - X[k][p] is added to z[p][k] with z laid out [Npoly][Mt] (DESIGN.md 7 item 22).
    The slave's loop indexes z[M p + k] there (sagecal_stochastic_slave.cpp:819-821), which with hybrid
    chunks sends the term of chunk k, term p to another slot; the test pins the Mt layout and shows that
    the two differ"""
    n8, Mt, M, Npoly, nsolbw = 8 * 2, 4, 3, 2, 1
    rng = np.random.default_rng(9)
    B = np.array([[1.0, 0.5]])
    rhok = np.full((nsolbw, Mt), 3.0)
    alphak = rng.uniform(0.5, 2.0, Mt)
    Bi = capi.consensus_prod_inverse_fed(B, rhok, alphak)
    J = rng.normal(0, 1, (nsolbw, Mt * n8))
    Y0 = rng.normal(0, 0.5, (nsolbw, Mt * n8))
    Zavg = rng.normal(0, 1, (Mt, Npoly, n8))
    X = rng.normal(0, 0.3, (Mt, Npoly, n8))

    def want(slot):
        Y = Y0.copy()
        Y[0] += np.repeat(rhok[0], n8) * J[0]
        z = (B[0][:, None] * Y[0][None, :]).reshape(-1)          # [Npoly][Mt][8N] flat
        for ci in range(Mt):
            for p in range(Npoly):
                s = slot(p, ci) * n8
                z[s:s + n8] += alphak[ci] * Zavg[ci, p] - X[ci, p]
        z = z.reshape(Npoly, Mt, n8)
        return np.einsum("kpq,qki->kpi", Bi, z)

    Y = Y0.copy()
    Z = np.zeros((Mt, Npoly, n8))
    rv, _, _, fb = capi.federated_bands_update(2, 1, np.ones(1), np.ones(1), J, B, Bi, rhok, alphak,
                                               Zavg, X, Y, Z)
    assert rv == 0 and not fb.any()
    mt_layout = want(lambda p, ci: Mt * p + ci)
    m_layout = want(lambda p, ci: M * p + ci)
    assert np.max(np.abs(Z - mt_layout)) <= 1e-13 * np.max(np.abs(mt_layout))
    assert np.max(np.abs(Z - m_layout)) > 1e-3
