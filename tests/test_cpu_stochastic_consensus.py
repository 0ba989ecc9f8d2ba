"""CPU tier of the consensus stochastic interval (sagecal -N -M -w -A, minibatch_consensus_mode.cpp:
450-672): include/dirac_b200_stochastic.h compiles on its own from a plain C99 host, which links and is
refused for no ADMM iterations and no polynomial terms; dirac_b200_consensus_bands_update, the host-only
ADMM step of one minibatch, against the driver's lines (:540-601) restated in numpy around the
reference's own update_global_z_multi, with B from setup_polynomials and Bi from find_prod_inverse_full.

The tests call the reference first and the product library afterwards, so that the reference's answers
can be recorded (tests/golden/ref/test_cpu_stochastic_consensus)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, MT = 5, 3          # stations, chunks (clusters' hybrid chunks summed)
RES_RATIO = 1.5       # minibatch_consensus_mode.cpp:262
CLM_DBL_MAX = 1e12    # Dirac_common.h
vp = C.c_void_p


@pytest.fixture(scope="module")
def capi():
    from sagecal_b200 import lib
    return lib.load()


def test_plain_c_host_compiles_links_and_is_refused(tmp_path):
    exe = os.path.join(str(tmp_path), "stochastic_consensus_caller")
    libdir = os.path.join(ROOT, "sagecal_b200")
    subprocess.check_call(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-Werror", "-o", exe,
                           os.path.join(ROOT, "tests", "c_caller", "stochastic_consensus_caller.c"),
                           "-I", os.path.join(ROOT, "include"), "-L", libdir, "-ldirac_b200", "-lm",
                           "-Wl,-rpath," + libdir])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "STOCHASTIC_CONSENSUS_CALLER OK" in out.stdout, (out.stdout, out.stderr)
    assert "nadmm = 0 ADMM iterations" in out.stderr and "Npoly = 0 polynomial terms" in out.stderr


def _p(a):
    return a.ctypes.data_as(vp)


def ref_basis(ref, Npoly, ffreq, freq0, ptype):
    """setup_polynomials over the bands' mean frequencies, as the driver calls it (:359): type 1 when
    Npoly is 1"""
    B = np.zeros((len(ffreq), Npoly))
    ref.lib.setup_polynomials.argtypes = [vp, C.c_int, C.c_int, vp, C.c_double, C.c_int]
    ref.lib.setup_polynomials(_p(B), Npoly, len(ffreq), _p(ffreq), freq0, 1 if Npoly == 1 else ptype)
    return B


def ref_prod_inverse(ref, B, rhok):
    nsolbw, Npoly = B.shape
    Bi = np.zeros((rhok.shape[1], Npoly, Npoly))
    ref.lib.find_prod_inverse_full.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int]
    ref.lib.find_prod_inverse_full(_p(B), _p(Bi), Npoly, nsolbw, rhok.shape[1], _p(rhok), 2)
    return Bi


def restated_update(ref, r00, r01, J, B, Bi, rhok, res_0, res_1, Y):
    """minibatch_consensus_mode.cpp:540-601 in numpy around the reference's update_global_z_multi;
    returns (res_0, res_1, fband, Y, Z)"""
    nsolbw, Npoly = B.shape
    n8 = 8 * N
    resband = np.zeros(nsolbw)
    for b in range(nsolbw):
        res_0 += r00[b]
        res_1 += r01[b]
        resband[b] = r01[b] if (r00[b] > 0.0 and r01[b] > 0.0) else CLM_DBL_MAX
    res_0 /= nsolbw
    res_1 /= nsolbw
    fband = (resband > RES_RATIO * res_1).astype(np.int32)
    Y = Y.copy()
    rho_i = np.repeat(rhok, n8, axis=1)            # [nsolbw, 8 N Mt]
    for b in range(nsolbw):
        if not fband[b]:
            Y[b] += rho_i[b] * J[b]
    z = B[0][:, None] * Y[0][None, :]             # [Npoly][Mt][8N]; band 0 whatever fband[0] says
    for b in range(1, nsolbw):
        if not fband[b]:
            z += B[b][:, None] * Y[b][None, :]
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


CASES = ["all-good", "middle-flagged", "band0-flagged", "nan-band"]


@pytest.mark.parametrize("Npoly", [1, 2, 3])
@pytest.mark.parametrize("case", CASES)
def test_bands_update_matches_the_driver(ref, capi, case, Npoly):
    nsolbw = 3
    rng = np.random.default_rng(100 + 10 * Npoly + CASES.index(case))
    m = 8 * N * MT
    ffreq = np.array([143e6, 151e6, 158e6])
    rhok = rng.uniform(2.0, 8.0, (nsolbw, MT))
    J = rng.normal(0, 1, (nsolbw, m))
    Y = rng.normal(0, 0.5, (nsolbw, m))
    r00 = rng.uniform(1.0, 2.0, nsolbw)
    r01 = rng.uniform(0.5, 0.9, nsolbw)
    res_0, res_1 = 1.3, 0.7                          # the running mixture of earlier minibatches
    if case == "middle-flagged":
        r01[1] = 10.0
    elif case == "band0-flagged":
        r01[0] = 10.0
    elif case == "nan-band":
        r00[2] = r01[2] = np.nan                      # a band without channels: 0 x 1/0
    B = ref_basis(ref, Npoly, ffreq, 150e6, 2)
    Bi = ref_prod_inverse(ref, B, rhok)
    w0, w1, wf, wY, wZ = restated_update(ref, r00, r01, J, B, Bi, rhok, res_0, res_1, Y)
    want_flags = {"all-good": [0, 0, 0], "middle-flagged": [0, 1, 0], "band0-flagged": [1, 0, 0],
                  "nan-band": [0, 0, 0]}[case]
    assert list(wf) == want_flags
    if case == "nan-band":
        assert np.isnan(w0) and np.isnan(w1)          # a NaN res_1 flags no band
    else:
        assert np.all(np.abs(np.where(r00 > 0, r01, CLM_DBL_MAX) - RES_RATIO * w1) > 1e-6)
    if case == "band0-flagged":
        assert np.array_equal(wY[0], Y[0])            # not updated, and still summed into z

    Yg = Y.copy()
    Zg = np.full((MT, Npoly, 8 * N), 123.0)           # overwritten: the driver keeps Z only for printing
    rv, g0, g1, gf = capi.consensus_bands_update(N, r00, r01, J, B, Bi, rhok, res_0, res_1, Yg, Zg)
    assert rv == 0
    assert list(gf) == list(wf)
    for g, w in ((g0, w0), (g1, w1)):
        assert (np.isnan(g) and np.isnan(w)) or abs(g - w) <= 1e-14 * abs(w)
    assert _close(Zg, wZ)
    assert _close(Yg, wY)
    if case == "band0-flagged":
        assert np.array_equal(Yg[0], Y[0])


def test_bands_update_refuses_empty_sizes(capi):
    """no bands or no polynomial terms: -1, nothing touched"""
    Y = np.ones((1, 8 * N * MT))
    Z = np.ones((MT, 1, 8 * N))
    for B in (np.ones((0, 1)), np.ones((1, 0))):
        rv, r0, r1, _ = capi.consensus_bands_update(N, np.ones(1), np.ones(1), Y, B,
                                                    np.ones((MT, 1, 1)), np.ones((1, MT)), 2.0, 3.0,
                                                    Y, Z)
        assert rv == -1 and (r0, r1) == (2.0, 3.0)
    assert (Y == 1).all() and (Z == 1).all()
