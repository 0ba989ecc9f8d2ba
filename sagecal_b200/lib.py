"""Loader for the product library `libdirac_b200.so` (hand-written sm_90a kernels behind the
Dirac C API).  There is no CPU fallback: a missing library or a missing GPU is an error."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .dirac_api import DiracAPI, SkyModel, baseline_t, clus_source_t, c_double_p, dptr, cptr  # noqa: F401

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdirac_b200.so")

#: every symbol include/dirac_b200.h declares
EXPORTED = [
    "sagefit_visibilities", "sagefit_visibilities_dual_pt_flt", "sagefit_visibilities_dual_pt",
    "sagefit_visibilities_dual_pt_one_gpu", "bfgsfit_visibilities", "bfgsfit_visibilities_gpu",
    "precalculate_coherencies", "predict_visibilities_multifreq", "generate_baselines",
    "preset_flags_and_data", "whiten_data", "dirac_b200_create", "dirac_b200_destroy", "dirac_b200_set_data",
    "dirac_b200_precalculate", "dirac_b200_get_coherencies", "dirac_b200_predict",
    "dirac_b200_grad", "dirac_b200_cost_window", "dirac_b200_grad_window", "dirac_b200_normal_eq",
    "dirac_b200_launch_count", "dirac_b200_sagefit",
    "dirac_b200_set_stream", "dirac_b200_profile_enable", "dirac_b200_profile_read",
    "dirac_b200_kernel_count", "dirac_b200_normal_eq_weighted", "dirac_b200_create_shard",
    "dirac_b200_set_comm", "dirac_b200_spd_solve", "dirac_b200_tri_solve", "dirac_b200_tri_solve_ld",
    "dirac_b200_set_option", "dirac_b200_nccl_unique_id", "dirac_b200_nccl_init",
    "dirac_b200_nccl_finalize", "dirac_b200_nccl_ready", "dirac_b200_comm_stats",
    "dirac_b200_noise_decisions", "dirac_b200_host_stats", "dirac_b200_consensus_basis",
    "dirac_b200_consensus_prod_inverse", "dirac_b200_consensus_step", "dirac_b200_sagefit_admm",
    "sagefit_visibilities_admm", "sagefit_visibilities_admm_dual_pt_flt",
    "calculate_residuals_multifreq", "dirac_b200_bigtri_solve", "dirac_b200_release_cache",
    "dirac_b200_sagefit_admm_rtr", "lbfgs_persist_init", "lbfgs_persist_clear",
    "lbfgs_persist_reset", "bfgsfit_minibatch_visibilities", "bfgsfit_minibatch_consensus",
    "precalculate_coherencies_withbeam", "precalculate_coherencies_withbeam_gpu",
    "predict_visibilities_multifreq_withbeam", "predict_visibilities_multifreq_withbeam_gpu",
    "calculate_residuals_multifreq_withbeam", "calculate_residuals_multifreq_withbeam_gpu",
    "dirac_b200_extract_phases", "precalculate_coherencies_multifreq",
    "precalculate_coherencies_multifreq_withbeam", "precalculate_coherencies_multifreq_withbeam_gpu",
    "bfgsfit_minibatch_visibilities_hbb", "bfgsfit_minibatch_consensus_hbb", "dirac_b200_barr_from_hbb",
]

#: every symbol include/dirac_b200_withsol.h declares (simulation with solutions)
WITHSOL_EXPORTED = [
    "predict_visibilities_multifreq_withsol", "predict_visibilities_multifreq_withsol_withbeam",
    "predict_visibilities_withsol_withbeam_gpu",
]

#: every symbol include/dirac_b200_diffuse.h declares (diffuse cluster from a spatial model)
DIFFUSE_EXPORTED = ["recalculate_diffuse_coherencies", "dirac_b200_diffuse_coherencies"]

#: every symbol include/dirac_b200_channels.h declares (per-channel refinement, driver option -b 1)
CHANNELS_EXPORTED = ["calculate_residuals", "dirac_b200_bfgsfit_channels", "dirac_b200_transfer_stats"]

#: every symbol include/dirac_b200_stochastic.h declares (stochastic calibration of an interval, with
#: or without spectral consensus over the bands)
STOCHASTIC_EXPORTED = ["dirac_b200_stochastic_interval", "dirac_b200_stochastic_consensus_interval",
                       "dirac_b200_consensus_bands_update", "dirac_b200_stochastic_interval_withbeam",
                       "dirac_b200_stochastic_consensus_interval_withbeam"]

#: every symbol include/dirac_b200_federated.h declares (federated stochastic calibration)
FEDERATED_EXPORTED = ["dirac_b200_stochastic_federated_interval", "calculate_manifold_average_projectback", "dirac_b200_manifold_projectback_dev",
                      "dirac_b200_consensus_prod_inverse_fed", "dirac_b200_federated_bands_update"]

#: every symbol include/dirac_b200_diagnostics.h declares (influence-function diagnostics, -i 1)
DIAGNOSTICS_EXPORTED = ["calculate_diagnostics_gpu"]


class DiracB200(DiracAPI):
    """The product library: the reference entry points (inherited bindings) plus the thin
    `dirac_b200_*` device layer."""

    def __init__(self, path: str = LIB_PATH):
        if not os.path.exists(path):
            raise RuntimeError(
                f"{path} not found: build it with `make -C sagecal_b200/csrc` (or "
                "`python -c 'import __graft_entry__ as g; g.build()'`). There is no CPU fallback.")
        super().__init__(path)
        L = self.lib
        vp = C.c_void_p
        i = C.c_int
        d = C.c_double
        dp = c_double_p
        L.dirac_b200_create.restype = vp
        L.dirac_b200_create.argtypes = [i, i, i, C.POINTER(baseline_t), C.POINTER(clus_source_t),
                                        i, i, dp, dp]
        L.dirac_b200_destroy.argtypes = [vp]
        L.dirac_b200_set_data.argtypes = [vp, dp]
        L.dirac_b200_precalculate.argtypes = [vp, dp, dp, dp, C.POINTER(clus_source_t), d, d, d, d,
                                              C.POINTER(baseline_t)]
        L.dirac_b200_get_coherencies.argtypes = [vp, dp]
        L.dirac_b200_predict.restype = d
        L.dirac_b200_predict.argtypes = [vp, dp, dp, i, i, d]
        L.dirac_b200_grad.argtypes = [vp, dp, dp, i, d]
        L.dirac_b200_cost_window.restype = d
        L.dirac_b200_cost_window.argtypes = [vp, dp, C.c_longlong, C.c_longlong, d]
        L.dirac_b200_grad_window.argtypes = [vp, dp, dp, C.c_longlong, C.c_longlong, d]
        L.dirac_b200_normal_eq.restype = d
        L.dirac_b200_normal_eq.argtypes = [vp, i, i, dp, dp, dp, dp]
        L.dirac_b200_normal_eq_weighted.restype = d
        L.dirac_b200_normal_eq_weighted.argtypes = [vp, i, i, dp, dp, dp, dp, dp]
        L.dirac_b200_launch_count.restype = C.c_ulonglong
        L.dirac_b200_sagefit.restype = i
        L.dirac_b200_sagefit.argtypes = [vp, dp, dp, i, i, i, i, i, i, d, d, i, dp, dp, dp]
        L.dirac_b200_set_stream.argtypes = [vp]
        L.dirac_b200_kernel_count.restype = C.c_ulonglong
        L.dirac_b200_kernel_count.argtypes = [i]
        L.dirac_b200_profile_enable.argtypes = [i]
        L.dirac_b200_profile_read.restype = i
        L.dirac_b200_profile_read.argtypes = [i, dp, dp]
        L.dirac_b200_set_option.restype = i
        L.dirac_b200_set_option.argtypes = [C.c_char_p, i]

    def set_option(self, name: str, value: int):
        if self.lib.dirac_b200_set_option(name.encode(), int(value)) != 0:
            raise KeyError(name)

    def host_stats(self, reset=False):
        """(host syncs, seconds blocked in them, collectives, collective bytes, seconds enqueueing them)"""
        n, c, b = C.c_ulonglong(0), C.c_ulonglong(0), C.c_ulonglong(0)
        w, e = C.c_double(0.0), C.c_double(0.0)
        self.lib.dirac_b200_host_stats(C.byref(n), C.byref(w), 1 if reset else 0)
        self.lib.dirac_b200_comm_stats(C.byref(c), C.byref(b), C.byref(e), 1 if reset else 0)
        return dict(host_syncs=n.value, host_wait_s=w.value, collectives=c.value,
                    collective_bytes=b.value, collective_enqueue_s=e.value)

    def transfer_stats(self, reset=False):
        """(sky models uploaded, bytes of coherencies copied between host and device)"""
        n, b = C.c_ulonglong(0), C.c_ulonglong(0)
        self.lib.dirac_b200_transfer_stats(C.byref(n), C.byref(b), 1 if reset else 0)
        return n.value, b.value

    def calculate_diagnostics_gpu(self, u, v, w, p, x, N, Nbase, tilesz, barr, sky, freqs, fdelta,
                                  beam=None, rho=None, Bpoly=None, Bi=None, Npoly=0, tdelta=10.0,
                                  dec0=1.0, Nt=4):
        """influence-function diagnostics (Dirac_radio.h:676).  x[chan][row][8]: data in; out: the
        eigenvalues of the four dR correlations in channel 0 of every timeslot, the residual in the
        other channels.  beam: a BeamSetup or None; rho [M], Bpoly [Npoly], Bi [M][Npoly][Npoly]: the
        consensus term (all three or none)"""
        L = self.lib
        d = C.c_double
        L.calculate_diagnostics_gpu.restype = C.c_int
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)
        rho, Bpoly, Bi = f64(rho), f64(Bpoly), f64(Bi)
        opt = lambda a: None if a is None else dptr(a)
        if beam is None:
            bhead = (0, d(0.0), d(0.0), d(0.0), d(0.0), d(0.0), None, None, None)
            btail = (None, None, None, None, None, 0)
        else:
            bhead, btail = beam.head(), beam.tail()
        return L.calculate_diagnostics_gpu(
            dptr(u), dptr(v), dptr(w), dptr(p), dptr(x), N, Nbase, tilesz, barr, sky.arr, sky.M,
            dptr(freqs), len(freqs), d(fdelta), d(tdelta), d(dec0), *bhead, *btail, opt(rho), opt(Bpoly),
            opt(Bi), sky.M, Npoly, len(freqs), Nt)

    def diagnostics_eval(self, N, Nbase, tilesz, barr, p, nchunk, coh, res, X):
        """the influence kernels of one cluster (dirac_b200_diagnostics_eval): coh, res [R][4] complex
        (channel 0), p [nchunk][N][8], X [4N][Nbase] complex.  returns (H [4N][4N] before the
        conditioning, AdV [4N][Nbase], dR [4][Nbase][Nbase], each complex), or None where refused"""
        L = self.lib
        L.dirac_b200_diagnostics_eval.restype = C.c_int
        L.dirac_b200_diagnostics_eval.argtypes = ([C.c_int] * 3 + [C.POINTER(baseline_t), c_double_p,
                                                   C.c_int] + [c_double_p] * 6)
        cf = lambda a: np.ascontiguousarray(a, dtype=np.complex128)
        n4 = 4 * N
        H = np.zeros((n4, n4), dtype=np.complex128, order="F")
        A = np.zeros((n4, Nbase), dtype=np.complex128, order="F")
        dR = np.zeros((4, Nbase, Nbase), dtype=np.complex128)
        Xf = np.asfortranarray(X, dtype=np.complex128)
        p = np.ascontiguousarray(p, dtype=np.float64)
        vp = lambda a: a.ctypes.data_as(c_double_p)
        rv = L.dirac_b200_diagnostics_eval(N, Nbase, tilesz, barr, dptr(p), nchunk, vp(cf(coh)),
                                           vp(cf(res)), vp(Xf), vp(H), vp(A), vp(dR))
        if rv != 0:
            return None
        # dR[c] is column major: element (row b, column bl) at bl*Nbase + b
        return H, A, np.ascontiguousarray(dR.transpose(0, 2, 1))

    def noise_decisions(self, reset=False) -> int:
        self.lib.dirac_b200_noise_decisions.restype = C.c_long
        return int(self.lib.dirac_b200_noise_decisions(1 if reset else 0))

    def launch_count(self) -> int:
        return int(self.lib.dirac_b200_launch_count())

    def lbfgs_direction(self, g, s, y, rho, npairs, next_):
        """one two-loop recursion of k_lbfgs_direction (dirac_b200_lbfgs_direction) on host vectors:
        g [m], s and y [Mmem, m], rho [Mmem], `npairs` valid pairs, `next_` the slot written next.
        returns pk = -H g [m], or None where the hook refuses the arguments"""
        L = self.lib
        L.dirac_b200_lbfgs_direction.restype = C.c_int
        L.dirac_b200_lbfgs_direction.argtypes = [C.c_int] * 4 + [c_double_p] * 5
        g = np.ascontiguousarray(g, dtype=np.float64)
        s = np.ascontiguousarray(s, dtype=np.float64)
        y = np.ascontiguousarray(y, dtype=np.float64)
        rho = np.ascontiguousarray(rho, dtype=np.float64)
        Mmem, m = s.shape
        assert y.shape == s.shape and g.shape == (m,) and rho.shape == (Mmem,)
        pk = np.zeros(m)
        rv = L.dirac_b200_lbfgs_direction(m, Mmem, npairs, next_, dptr(g), dptr(s), dptr(y),
                                          dptr(rho), dptr(pk))
        return None if rv != 0 else pk

    def lbfgs_step_update(self, alpha, xk, pk, gk_old, gk_new, rho, ci):
        """k_lbfgs_step then k_lbfgs_update into slot ci of rho (dirac_b200_lbfgs_step_update).
        returns dict(xk1, sk, yk, rho, gg = ||gk_new||^2, xk = xk after the update)"""
        L = self.lib
        L.dirac_b200_lbfgs_step_update.restype = C.c_int
        L.dirac_b200_lbfgs_step_update.argtypes = ([C.c_int, C.c_double] + [c_double_p] * 4
                                                   + [C.c_int, C.c_int] + [c_double_p] * 7)
        a = [np.ascontiguousarray(v, dtype=np.float64) for v in (xk, pk, gk_old, gk_new, rho)]
        m, Mmem = len(a[0]), len(a[4])
        out = dict(xk1=np.zeros(m), sk=np.zeros(m), yk=np.zeros(m), rho=np.zeros(Mmem),
                   gg=np.zeros(1), xk=np.zeros(m))
        rv = L.dirac_b200_lbfgs_step_update(m, alpha, *[dptr(v) for v in a[:4]], Mmem, ci,
                                            dptr(a[4]), *[dptr(out[k]) for k in
                                                          ("xk1", "sk", "yk", "rho", "gg", "xk")])
        assert rv == 0
        out["gg"] = float(out["gg"][0])
        return out

    def lbfgs_nrm2(self, g):
        """||g||^2 of k_lbfgs_nrm2 (dirac_b200_lbfgs_nrm2)"""
        L = self.lib
        L.dirac_b200_lbfgs_nrm2.restype = C.c_double
        L.dirac_b200_lbfgs_nrm2.argtypes = [C.c_int, c_double_p]
        g = np.ascontiguousarray(g, dtype=np.float64)
        return float(L.dirac_b200_lbfgs_nrm2(len(g), dptr(g)))

    def band_eval(self, N, Nbase, tilesz, barr, sky: SkyModel, coh, x, Nf, P, nu, maxnc=None,
                  Y=None, Z=None, rho=None):
        """the minibatch band passes (dirac_b200_band_eval): one band of Nf channels, coh
        [Nf][row][M][4] complex and x [Nf][row][8], staged as bfgsfit_minibatch_visibilities stages
        it, in a band state of capacity maxnc (default Nf); the Jones vectors P [npts, 8 N Mt]
        evaluated in order with the fits' cost and gradient (consensus terms with Y, Z, rho).
        returns dict(cost [npts], grad [npts, 8 N Mt], res [Nf * row * 8]: residual of the last
        point), or None where the hook refuses the arguments"""
        L = self.lib
        L.dirac_b200_band_eval.restype = C.c_int
        L.dirac_b200_band_eval.argtypes = ([C.c_int] * 3 + [C.POINTER(baseline_t),
                                           C.POINTER(clus_source_t)] + [C.c_int] * 2
                                           + [c_double_p] * 2 + [C.c_int] * 3 + [c_double_p] * 4
                                           + [C.c_double] + [c_double_p] * 3)
        P = np.ascontiguousarray(np.atleast_2d(P), dtype=np.float64)
        coh = np.ascontiguousarray(coh, dtype=np.complex128)
        x = np.ascontiguousarray(x, dtype=np.float64)
        cons = [None if v is None else np.ascontiguousarray(v, dtype=np.float64) for v in (Y, Z, rho)]
        npts = P.shape[0]
        cost = np.zeros(max(npts, 1))
        grad = np.zeros((max(npts, 1), P.shape[1]))
        res = np.zeros(8 * Nbase * tilesz * max(Nf, 1))
        rv = L.dirac_b200_band_eval(N, Nbase, tilesz, barr, sky.arr, sky.M, sky.Mt,
                                    cptr(coh), dptr(x), Nf,
                                    Nf if maxnc is None else maxnc, npts, dptr(P),
                                    *[dptr(v) if v is not None else None for v in cons], nu,
                                    dptr(cost), dptr(grad.reshape(-1)), dptr(res))
        if rv != 0:
            return None
        return dict(cost=cost, grad=grad, res=res[:8 * Nbase * tilesz * Nf])

    def kernel_count(self, kind) -> int:
        return int(self.lib.dirac_b200_kernel_count(kind))

    def set_stream(self, cuda_stream_ptr):
        self.lib.dirac_b200_set_stream(C.c_void_p(cuda_stream_ptr))

    def profile_enable(self, on=True):
        self.lib.dirac_b200_profile_enable(1 if on else 0)

    def profile_read(self, kind):
        """(launches, total ms, total algorithmic bytes) of the recorded launches of `kind`"""
        ms = C.c_double(0.0)
        by = C.c_double(0.0)
        n = self.lib.dirac_b200_profile_read(kind, C.byref(ms), C.byref(by))
        return n, ms.value, by.value


class DeviceProblem:
    """One solve interval resident on the GPU (dirac_b200_create ... dirac_b200_destroy)."""

    def __init__(self, api: DiracB200, N, Nbase, tilesz, barr, sky: SkyModel, coh, x):
        self.api = api
        self.N, self.Nbase, self.tilesz, self.sky = N, Nbase, tilesz, sky
        self.n = 8 * Nbase * tilesz
        self.m = 8 * N * sky.Mt
        self.h = api.lib.dirac_b200_create(N, Nbase, tilesz, barr, sky.arr, sky.M, sky.Mt,
                                           cptr(coh) if coh is not None else None,
                                           dptr(x) if x is not None else None)
        if not self.h:
            raise RuntimeError("dirac_b200_create failed")

    def close(self):
        if self.h:
            self.api.lib.dirac_b200_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def set_data(self, x):
        self.api.lib.dirac_b200_set_data(self.h, dptr(x))

    def precalculate(self, u, v, w, freq0, fdelta, uvmin=0.0, uvmax=1e9, barr=None):
        self.api.lib.dirac_b200_precalculate(self.h, dptr(u), dptr(v), dptr(w), self.sky.arr,
                                             freq0, fdelta, uvmin, uvmax, barr)

    def diffuse_coherencies(self, u, v, w, freq0, fdelta, cid, sh_n0, sh_beta, Z):
        """dirac_b200_diffuse_coherencies: rewrite local cluster cid's resident coherencies from the
        spatial model Z (2N x 2G complex, column major, G = sh_n0^2)"""
        L = self.api.lib
        L.dirac_b200_diffuse_coherencies.restype = C.c_int
        L.dirac_b200_diffuse_coherencies.argtypes = [C.c_void_p, c_double_p, c_double_p, c_double_p,
                                                     C.POINTER(clus_source_t), C.c_double, C.c_double,
                                                     C.c_int, C.c_int, C.c_double, c_double_p]
        Zf = np.asfortranarray(Z, dtype=np.complex128).reshape(-1, order="F")
        return L.dirac_b200_diffuse_coherencies(self.h, dptr(u), dptr(v), dptr(w), self.sky.arr, freq0,
                                                fdelta, cid, sh_n0, sh_beta, cptr(Zf))

    def get_coherencies(self):
        coh = np.zeros(4 * self.sky.M * self.Nbase * self.tilesz, dtype=np.complex128)
        self.api.lib.dirac_b200_get_coherencies(self.h, cptr(coh))
        return coh

    def predict(self, pp, out_mode=2, cost_mode=0, nu=0.0):
        """returns (cost, out) — out is the model (2) or residual (1) in API layout."""
        out = np.zeros(self.n) if out_mode else None
        c = self.api.lib.dirac_b200_predict(self.h, dptr(pp), dptr(out) if out_mode else None,
                                            out_mode, cost_mode, nu)
        return c, out

    def cost(self, pp, robust=False, nu=0.0):
        return self.api.lib.dirac_b200_predict(self.h, dptr(pp), None, 0, 2 if robust else 1, nu)

    def grad(self, pp, robust=False, nu=0.0):
        g = np.zeros(self.m)
        self.api.lib.dirac_b200_grad(self.h, dptr(pp), dptr(g), 1 if robust else 0, nu)
        return g

    def cost_window(self, pp, row0, nrows, nu):
        """Student's-t cost of the rows [row0, row0 + nrows) alone"""
        return self.api.lib.dirac_b200_cost_window(self.h, dptr(pp), row0, nrows, nu)

    def grad_window(self, pp, row0, nrows, nu):
        """gradient of cost_window with the reference's minibatch sign (minus the true gradient)"""
        g = np.zeros(self.m)
        self.api.lib.dirac_b200_grad_window(self.h, dptr(pp), dptr(g), row0, nrows, nu)
        return g

    def sagefit(self, pp, x_out=None, max_emiter=3, max_iter=2, max_lbfgs=10, lbfgs_m=7, linsolv=0,
                solver_mode=1, nulow=2.0, nuhigh=30.0, randomize=0):
        """dirac_b200_sagefit on the resident problem; pp updated in place.
        returns (retval, mean_nu, res_0, res_1)"""
        nu, r0, r1 = C.c_double(0.0), C.c_double(0.0), C.c_double(0.0)
        rv = self.api.lib.dirac_b200_sagefit(self.h, dptr(pp),
                                             dptr(x_out) if x_out is not None else None,
                                             max_emiter, max_iter, max_lbfgs, lbfgs_m, linsolv,
                                             solver_mode, nulow, nuhigh, randomize, C.byref(nu),
                                             C.byref(r0), C.byref(r1))
        return rv, nu.value, r0.value, r1.value

    def line_model(self, xk, pk, alphas, nu, alpha_res):
        """the LBFGS line model along pk from xk as one iteration sets it up (dirac_b200_line_model).
        returns dict(E0, E1, E2 [API layout], poly [5], cost_gauss, cost_robust [per alpha],
        res [line residual at alpha_res], shape (TB, NST, WARPS) of the k_stream_all<1> launch)"""
        L = self.api.lib
        L.dirac_b200_line_model.restype = None
        L.dirac_b200_line_model.argtypes = [C.c_void_p, c_double_p, c_double_p, C.c_int, c_double_p,
                                            C.c_double, C.c_double, c_double_p, c_double_p, c_double_p,
                                            c_double_p, C.POINTER(C.c_int)]
        xk = np.ascontiguousarray(xk, dtype=np.float64)
        pk = np.ascontiguousarray(pk, dtype=np.float64)
        alphas = np.ascontiguousarray(alphas, dtype=np.float64)
        E = np.zeros(3 * self.n)
        poly = np.zeros(5)
        costs = np.zeros(2 * len(alphas))
        res = np.zeros(self.n)
        shape = (C.c_int * 3)()
        L.dirac_b200_line_model(self.h, dptr(xk), dptr(pk), len(alphas), dptr(alphas), nu, alpha_res,
                                dptr(E), dptr(poly), dptr(costs), dptr(res), shape)
        return dict(E0=E[:self.n], E1=E[self.n:2 * self.n], E2=E[2 * self.n:], poly=poly,
                    cost_gauss=costs[0::2], cost_robust=costs[1::2], res=res, shape=tuple(shape))

    #: operation bits of one rtr_eval evaluation (rtr.cu: RTR_HOOK_*)
    RTR_COST, RTR_VEC, RTR_COUNTS, RTR_ETA, RTR_UNIT = 1, 2, 4, 8, 16

    def lbfgs_trace(self, pp, itmax, M, robust=False, nu=2.0):
        """LBFGS on the resident data from pp as bfgsfit runs it, traced (dirac_b200_lbfgs_trace).
        returns dict(p [final], niter, alphak, ncost, slot, gnorm [per iteration], iterates
        [niter, m]), or None where the memory size M cannot be held"""
        L = self.api.lib
        L.dirac_b200_lbfgs_trace.restype = C.c_int
        L.dirac_b200_lbfgs_trace.argtypes = [C.c_void_p, c_double_p, C.c_int, C.c_int, C.c_int,
                                             C.c_double, c_double_p, C.POINTER(C.c_longlong),
                                             C.POINTER(C.c_int), c_double_p, c_double_p]
        p = np.array(pp, dtype=np.float64)
        n = max(itmax, 1)
        alphak, gnorm = np.zeros(n), np.zeros(n)
        ncost = np.zeros(n, dtype=np.int64)
        slot = np.zeros(n, dtype=np.int32)
        it = np.zeros((n, self.m))
        k = L.dirac_b200_lbfgs_trace(self.h, dptr(p), itmax, M, int(robust), nu, dptr(alphak),
                                     ncost.ctypes.data_as(C.POINTER(C.c_longlong)),
                                     slot.ctypes.data_as(C.POINTER(C.c_int)), dptr(gnorm),
                                     dptr(it.reshape(-1)))
        if k < 0:
            return None
        return dict(p=p, niter=k, alphak=alphak[:k], ncost=ncost[:k], slot=slot[:k],
                    gnorm=gnorm[:k], iterates=it[:k])

    def rtr_eval(self, k, ck, evals, xw=None, nu=2.0, keep=True, force_device=False):
        """the RTR device evaluator of cluster k, chunk ck on the data vector as hidden data
        (dirac_b200_rtr_eval): one condensation (unit weights, or Student's-t weights at xw with nu;
        keep=False condenses the scalars only), then `evals` in order, each a dict with x [8N] and
        optional eta [8N], cost / vec / counts / unit (unit_weights() first) flags.
        returns dict(results=[dict(cost, vec, counts) per evaluation, None where not asked],
        slw [sum(log w - w) / rows], nslice, tslice, inline)"""
        L = self.api.lib
        L.dirac_b200_rtr_eval.restype = None
        L.dirac_b200_rtr_eval.argtypes = [C.c_void_p, C.c_int, C.c_int, c_double_p, C.c_double,
                                          C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), c_double_p,
                                          c_double_p, c_double_p, c_double_p, c_double_p, c_double_p]
        n8, ne = 8 * self.N, len(evals)
        ops = np.zeros(ne, dtype=np.int32)
        X = np.zeros((ne, n8))
        ETA = np.zeros((ne, n8))
        for i, e in enumerate(evals):
            X[i] = e["x"]
            if e.get("eta") is not None:
                ETA[i] = e["eta"]
                ops[i] |= self.RTR_ETA
            ops[i] |= ((self.RTR_COST if e.get("cost") else 0) | (self.RTR_VEC if e.get("vec") else 0)
                       | (self.RTR_COUNTS if e.get("counts") else 0)
                       | (self.RTR_UNIT if e.get("unit") else 0))
        cost = np.zeros(ne)
        vec = np.zeros((ne, n8))
        cnt = np.zeros((ne, self.N))
        info = np.zeros(4)
        xw_arr = None if xw is None else np.ascontiguousarray(xw, dtype=np.float64)
        L.dirac_b200_rtr_eval(self.h, k, ck, dptr(xw_arr) if xw_arr is not None else None, nu,
                              1 if keep else 0, 1 if force_device else 0, ne,
                              ops.ctypes.data_as(C.POINTER(C.c_int)), dptr(X), dptr(ETA), dptr(cost),
                              dptr(vec), dptr(cnt), dptr(info))
        res = [dict(cost=cost[i] if ops[i] & self.RTR_COST else None,
                    vec=vec[i] if ops[i] & self.RTR_VEC else None,
                    counts=cnt[i] if ops[i] & self.RTR_COUNTS else None) for i in range(ne)]
        return dict(results=res, slw=info[0], nslice=int(info[1]), tslice=int(info[2]),
                    inline=bool(info[3]))

    def os_normal_eq(self, clus, chunk, l, pblk, xd, wt=None):
        """J^T J and J^T e of ordered subset l as the OS-LM forms them (dirac_b200_os_normal_eq), on
        hidden data xd with sqrt-weights wt (API layout, full interval) or none.
        returns (JTJ, JTe, path dict(misaligned, s0, s1, nJ))"""
        L = self.api.lib
        L.dirac_b200_os_normal_eq.restype = None
        L.dirac_b200_os_normal_eq.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, c_double_p,
                                              c_double_p, c_double_p, c_double_p, c_double_p,
                                              C.POINTER(C.c_longlong)]
        n8 = 8 * self.N
        JTJ = np.zeros((n8, n8))
        JTe = np.zeros(n8)
        path = (C.c_longlong * 4)()
        pblk = np.ascontiguousarray(pblk, dtype=np.float64)
        xd = np.ascontiguousarray(xd, dtype=np.float64)
        wt = None if wt is None else np.ascontiguousarray(wt, dtype=np.float64)
        L.dirac_b200_os_normal_eq(self.h, clus, chunk, l, dptr(pblk), dptr(xd),
                                  dptr(wt) if wt is not None else None, dptr(JTJ.reshape(-1)),
                                  dptr(JTe), path)
        return JTJ, JTe, dict(misaligned=bool(path[0]), s0=int(path[1]), s1=int(path[2]),
                              nJ=int(path[3]))

    def irls_update(self, clus, chunk, pblk, xd, wt, nu0, nulow=2.0, nuhigh=30.0):
        """the update between two robust-LM rounds (dirac_b200_irls_update): residual at pblk of the
        hidden data xd, weights from wt (API layout, full interval) with nu0.
        returns (new weights [rows outside the chunk as given], lambda, sumq, nu)"""
        L = self.api.lib
        L.dirac_b200_irls_update.restype = None
        L.dirac_b200_irls_update.argtypes = [C.c_void_p, C.c_int, C.c_int, c_double_p, c_double_p,
                                             c_double_p, C.c_double, C.c_double, C.c_double,
                                             c_double_p]
        w = np.array(wt, dtype=np.float64)
        out3 = np.zeros(3)
        L.dirac_b200_irls_update(self.h, clus, chunk,
                                 dptr(np.ascontiguousarray(pblk, dtype=np.float64)),
                                 dptr(np.ascontiguousarray(xd, dtype=np.float64)), dptr(w), nu0,
                                 nulow, nuhigh, dptr(out3))
        return w, out3[0], out3[1], out3[2]

    def lm_chunk(self, clus, chunk, pblk, xd, itmax, opts=None, linsolv=0, os_=False, robust=False,
                 nulow=2.0, nuhigh=30.0, nu0=2.0):
        """LM (clevmar / oslevmar) or robust LM (rlevmar / osrlevmar) of one chunk on hidden data xd,
        through the solvers' own chunk functions (dirac_b200_lm_chunk).
        returns (pblk, info [10], nu)"""
        L = self.api.lib
        L.dirac_b200_lm_chunk.restype = None
        L.dirac_b200_lm_chunk.argtypes = [C.c_void_p, C.c_int, C.c_int, c_double_p, c_double_p,
                                          C.c_int, c_double_p, C.c_int, C.c_int, C.c_int, C.c_double,
                                          C.c_double, C.POINTER(C.c_double), c_double_p]
        p = np.array(pblk, dtype=np.float64)
        info = np.zeros(10)
        nu = C.c_double(nu0)
        o = None if opts is None else np.ascontiguousarray(opts, dtype=np.float64)
        L.dirac_b200_lm_chunk(self.h, clus, chunk, dptr(p),
                              dptr(np.ascontiguousarray(xd, dtype=np.float64)), itmax,
                              dptr(o) if o is not None else None, linsolv, int(os_), int(robust),
                              nulow, nuhigh, C.byref(nu), dptr(info))
        return p, info, nu.value

    #: kernel a cluster pass ran (internal.cuh: DB_CP_*); "none": the chunk has no timeslot
    CLUSTER_PASS_KERNELS = ("lin", "lin_grad", "split", "tile", "none")

    def cluster_pass(self, clus, chunk, mode, pblk, x, write_out=True, with_jte=False,
                     form_hidden=False, beta=1.0, pblk_old=None, wt=None, out_init=None,
                     inplace=False):
        """one streaming pass of chunk `chunk` of cluster clus through the LM visits' dispatch
        (dirac_b200_cluster_pass_eval): mode 0 INIT, 1 TRIAL, 2 ADD, 3 SUB, 4 GIVEN; input x, weights
        wt and the output vector's initial content out_init (default 0) in API layout, full interval;
        inplace: the output vector is the input vector.
        returns dict(kernel, out [all rows], jte [8N], cost); kernel None (out, jte, cost NaN, as the
        hook leaves them) where the hook refuses the arguments"""
        L = self.api.lib
        L.dirac_b200_cluster_pass_eval.restype = C.c_int
        L.dirac_b200_cluster_pass_eval.argtypes = ([C.c_void_p] + [C.c_int] * 6 + [C.c_double]
                                                   + [c_double_p] * 5 + [C.c_int] + [c_double_p] * 3)
        f64 = lambda v: None if v is None else np.ascontiguousarray(v, dtype=np.float64)
        pblk, pblk_old, x, wt = f64(pblk), f64(pblk_old), f64(x), f64(wt)
        out_init = np.zeros(self.n) if out_init is None else f64(out_init)
        out = np.full(self.n, np.nan)
        jte = np.full(8 * self.N, np.nan)
        cost = np.full(1, np.nan)
        opt = lambda v: dptr(v) if v is not None else None
        k = L.dirac_b200_cluster_pass_eval(self.h, clus, chunk, mode, int(write_out), int(with_jte),
                                           int(form_hidden), beta, dptr(pblk), opt(pblk_old),
                                           dptr(x), opt(wt), dptr(out_init), int(inplace),
                                           dptr(out), dptr(jte), dptr(cost))
        return dict(kernel=None if k < 0 else self.CLUSTER_PASS_KERNELS[k], out=out, jte=jte,
                    cost=float(cost[0]))

    def cluster_hidden(self, clus, sign, beta, pp, r, dh):
        """the row-mapped add (sign > 0) or subtract (sign < 0) of cluster clus's model at the Jones
        pp [8 N Mt] (dirac_b200_cluster_hidden_eval) on the residual r and the hidden data dh (API
        layout).  returns the vector it writes (hidden data, or residual), or None where refused"""
        L = self.api.lib
        L.dirac_b200_cluster_hidden_eval.restype = C.c_int
        L.dirac_b200_cluster_hidden_eval.argtypes = ([C.c_void_p, C.c_int, C.c_int, C.c_double]
                                                     + [c_double_p] * 4)
        f64 = lambda v: np.ascontiguousarray(v, dtype=np.float64)
        out = np.full(self.n, np.nan)
        rv = L.dirac_b200_cluster_hidden_eval(self.h, clus, sign, beta, dptr(f64(pp)), dptr(f64(r)),
                                              dptr(f64(dh)), dptr(out))
        return None if rv != 0 else out

    def normal_eq(self, clus, chunk, pblk, xd):
        n8 = 8 * self.N
        JTJ = np.zeros((n8, n8))
        JTe = np.zeros(n8)
        pblk = np.ascontiguousarray(pblk, dtype=np.float64)
        c = self.api.lib.dirac_b200_normal_eq(self.h, clus, chunk, dptr(pblk), dptr(xd),
                                              dptr(JTJ.reshape(-1)), dptr(JTe))
        return c, JTJ, JTe

    def normal_eq_weighted(self, clus, chunk, pblk, xd, wt):
        n8 = 8 * self.N
        JTJ = np.zeros((n8, n8))
        JTe = np.zeros(n8)
        pblk = np.ascontiguousarray(pblk, dtype=np.float64)
        c = self.api.lib.dirac_b200_normal_eq_weighted(self.h, clus, chunk, dptr(pblk), dptr(xd),
                                                       dptr(wt), dptr(JTJ.reshape(-1)), dptr(JTe))
        return c, JTJ, JTe


_api = None


def load() -> DiracB200:
    global _api
    if _api is None:
        _api = DiracB200()
    return _api
