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
    "dirac_b200_grad", "dirac_b200_normal_eq", "dirac_b200_launch_count", "dirac_b200_sagefit",
    "dirac_b200_set_stream", "dirac_b200_profile_enable", "dirac_b200_profile_read",
    "dirac_b200_kernel_count", "dirac_b200_normal_eq_weighted", "dirac_b200_create_shard",
    "dirac_b200_set_comm", "dirac_b200_spd_solve", "dirac_b200_tri_solve",
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

    def noise_decisions(self, reset=False) -> int:
        self.lib.dirac_b200_noise_decisions.restype = C.c_long
        return int(self.lib.dirac_b200_noise_decisions(1 if reset else 0))

    def launch_count(self) -> int:
        return int(self.lib.dirac_b200_launch_count())

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
