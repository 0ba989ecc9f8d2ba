"""TEST INFRASTRUCTURE ONLY.  ctypes access to the CPU restatement (oracle/liboracle.so, built from
oracle/dirac_oracle.c).  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may
import this module; the product package never does."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORC_PATH = os.path.join(_HERE, "liboracle.so")
RTR_PATH = os.path.join(_HERE, "librtr_harness.so")
RTR_TENSOR_PATH = os.path.join(_HERE, "librtr_tensor_check.so")

dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int)
up = C.POINTER(C.c_ubyte)


class orc_problem(C.Structure):
    _fields_ = [("N", C.c_int), ("Nbase", C.c_int), ("tilesz", C.c_int), ("M", C.c_int),
                ("Mt", C.c_int), ("sta1", ip), ("sta2", ip), ("flag", up), ("nchunk", ip),
                ("chunk0", ip), ("chunk_off", ip), ("coh", dp)]


class orc_sky(C.Structure):
    _fields_ = [("M", C.c_int), ("src0", ip)] + [(n, dp) for n in
                ("ll", "mm", "nn", "sI", "sQ", "sU", "sV")] + [("stype", up), ("gauss", dp)] + \
               [(n, dp) for n in ("sI0", "sQ0", "sU0", "sV0", "f0", "spec_idx", "spec_idx1",
                                  "spec_idx2")]


class orc_lbfgs_trace(C.Structure):
    _fields_ = [("alphak", dp), ("ncost", C.POINTER(C.c_longlong)), ("slot", ip), ("gnorm", dp),
                ("iterates", dp), ("niter", C.c_int), ("margin", C.c_double)]


def mult_hessian(g, s, y, rho, npairs, next_):
    """orc_mult_hessian: H g of the two-loop recursion (without the sign of the search direction)
    from s, y [Mmem, m], rho [Mmem], `npairs` valid pairs and `next_` the slot written next"""
    L = C.CDLL(ORC_PATH)
    L.orc_mult_hessian.argtypes = [C.c_int, dp, dp, dp, dp, dp, C.c_int, C.c_int]
    g, s, y, rho = (np.ascontiguousarray(a, dtype=np.float64) for a in (g, s, y, rho))
    pk = np.zeros(len(g))
    L.orc_mult_hessian(len(g), _d(pk), _d(g), _d(s), _d(y), _d(rho), npairs, next_)
    return pk


def available():
    return os.path.exists(ORC_PATH)


def _d(a):
    return a.ctypes.data_as(dp)


class Oracle:
    """the restated hot path bound to one synthetic problem (sagecal_b200.synth.Problem)"""

    def __init__(self, pr, coh=None, flag=None):
        L = C.CDLL(ORC_PATH, mode=C.RTLD_GLOBAL)
        self.L = L
        # RTR / RSD / NSD control flow on the oracle's evaluators (registers itself with liboracle
        # when loaded: orc_sagefit then accepts solver_mode 4-6)
        self.H = C.CDLL(RTR_PATH) if os.path.exists(RTR_PATH) else None
        self.pr = pr
        d, i = C.c_double, C.c_int
        pp = C.POINTER(orc_problem)
        L.orc_predict_full.argtypes = [pp, dp, dp]
        L.orc_predict_cluster.argtypes = [pp, i, dp, dp]
        L.orc_predict_chunk.argtypes = [pp, i, i, i, dp, dp]
        L.orc_cost.restype = d
        L.orc_cost.argtypes = [pp, dp, dp, i, d]
        L.orc_grad.argtypes = [pp, dp, dp, dp, i, d]
        L.orc_normal_eq.restype = d
        L.orc_normal_eq.argtypes = [pp, i, i, i, dp, dp, dp, dp, dp]
        L.orc_normal_eq_os.restype = None
        L.orc_normal_eq_os.argtypes = [pp, i, i, i, dp, dp, dp, i, dp, dp]
        L.orc_lm_chunk.argtypes = [pp, i, i, i, dp, dp, i, dp, i, i, dp]
        L.orc_rlm_chunk.argtypes = [pp, i, i, i, dp, dp, i, i, i, d, d, dp, dp]
        L.orc_update_w_and_nu.restype = d
        L.orc_update_w_and_nu.argtypes = [d, dp, dp, i, d, d]
        L.orc_lbfgs.argtypes = [pp, dp, dp, i, i, i, d]
        L.orc_mult_hessian.argtypes = [i, dp, dp, dp, dp, dp, i, i]
        L.orc_lbfgs_traced.argtypes = [pp, dp, dp, i, i, i, d, C.POINTER(orc_lbfgs_trace)]
        L.orc_lbfgs_last_margin.restype = d
        L.orc_noise_decisions.restype = C.c_long
        L.orc_noise_decisions.argtypes = [i]
        L.orc_sagefit.restype = i
        L.orc_sagefit.argtypes = [pp, dp, dp, i, i, i, i, i, i, d, d, dp, dp, dp]
        L.orc_bfgsfit.restype = i
        L.orc_bfgsfit.argtypes = [pp, dp, dp, i, i, i, d, dp, dp]
        if self.H is not None:
            self.H.harness_rtr_solve_admm.argtypes = [pp, i, i, i, i, i, dp, i, dp, i, i, d, d, dp, dp,
                                                      i, dp, dp, d]
            self.H.harness_rtr_solve_admm.restype = None
        # the arithmetic of the product's RTR kernels (rtr_math.cuh) on the CPU
        self.HT = C.CDLL(RTR_TENSOR_PATH) if os.path.exists(RTR_TENSOR_PATH) else None
        if self.HT is not None:
            self.HT.harness_rtr_solve_tensor.argtypes = [pp, i, i, i, dp, i, dp, i, i, d, d, dp, dp,
                                                         i, dp, dp, d]
            self.HT.harness_rtr_solve_tensor.restype = None
        L.orc_rtr_raw.restype = d
        L.orc_rtr_raw.argtypes = [pp, i, i, i, dp, dp, dp, dp, dp]
        L.orc_rtr_counts.argtypes = [pp, i, i, dp]
        L.orc_rtr_weights.restype = d
        L.orc_rtr_weights.argtypes = [pp, i, i, i, dp, dp, d, dp]
        L.orc_generate_baselines.argtypes = [i, i, i, ip, ip]
        L.orc_preset_flags_and_data.argtypes = [i, dp, up, dp]
        ps = C.POINTER(orc_sky)
        L.orc_coherencies.argtypes = [ps, dp, dp, dp, i, d, d, d, d, up, dp]
        L.orc_predict_multifreq.argtypes = [ps, dp, dp, dp, i, dp, i, d, i, dp]
        # problem arrays
        self.sta1 = np.ascontiguousarray(pr.sta1, dtype=np.int32)
        self.sta2 = np.ascontiguousarray(pr.sta2, dtype=np.int32)
        self.flag = np.ascontiguousarray(pr.flag if flag is None else flag, dtype=np.uint8)
        self.nchunk = np.ascontiguousarray(pr.nchunk, dtype=np.int32)
        self.chunk0 = np.concatenate([[0], np.cumsum(self.nchunk)[:-1]]).astype(np.int32)
        self.chunk_off = (np.arange(pr.Mt) * 8 * pr.N).astype(np.int32)
        self.coh = np.ascontiguousarray(pr.coh if coh is None else coh)
        P = orc_problem()
        P.N, P.Nbase, P.tilesz, P.M, P.Mt = pr.N, pr.Nbase, pr.tilesz, pr.M, pr.Mt
        P.sta1 = self.sta1.ctypes.data_as(ip)
        P.sta2 = self.sta2.ctypes.data_as(ip)
        P.flag = self.flag.ctypes.data_as(up)
        P.nchunk = self.nchunk.ctypes.data_as(ip)
        P.chunk0 = self.chunk0.ctypes.data_as(ip)
        P.chunk_off = self.chunk_off.ctypes.data_as(ip)
        P.coh = self.coh.view(np.float64).ctypes.data_as(dp) if self.coh is not None else None
        self.P = P
        self.n = 8 * pr.Nbase1
        self.m = 8 * pr.N * pr.Mt

    # ---- passes ----
    def predict_full(self, pp):
        out = np.zeros(self.n)
        self.L.orc_predict_full(C.byref(self.P), _d(pp), _d(out))
        return out

    def predict_cluster(self, k, pp):
        out = np.zeros(self.n)
        self.L.orc_predict_cluster(C.byref(self.P), k, _d(pp), _d(out))
        return out

    def predict_chunk(self, k, t0, ntiles, pblk):
        """model of cluster k with one parameter block over tiles [t0, t0 + ntiles)"""
        out = np.zeros(8 * ntiles * self.pr.Nbase)
        self.L.orc_predict_chunk(C.byref(self.P), k, t0, ntiles,
                                 _d(np.ascontiguousarray(pblk, dtype=np.float64)), _d(out))
        return out

    def cost(self, pp, x, robust=False, nu=2.0):
        return self.L.orc_cost(C.byref(self.P), _d(pp), _d(x), int(robust), nu)

    def grad(self, pp, x, robust=False, nu=2.0):
        g = np.zeros(self.m)
        self.L.orc_grad(C.byref(self.P), _d(pp), _d(x), _d(g), int(robust), nu)
        return g

    def chunk_tiles(self, k, ck):
        nch = int(self.nchunk[k])
        tc = (self.pr.tilesz + nch - 1) // nch
        t0 = min(ck * tc, self.pr.tilesz)
        return t0, min(t0 + tc, self.pr.tilesz) - t0

    def normal_eq(self, k, t0, ntiles, pblk, xd, wt=None):
        n8 = 8 * self.pr.N
        JTJ = np.zeros((n8, n8))
        JTe = np.zeros(n8)
        pblk = np.ascontiguousarray(pblk)
        xd = np.ascontiguousarray(xd)
        c = self.L.orc_normal_eq(C.byref(self.P), k, t0, ntiles, _d(pblk), _d(xd),
                                 _d(wt) if wt is not None else None, _d(JTJ.reshape(-1)), _d(JTe))
        return c, JTJ, JTe

    def normal_eq_os(self, k, t0, ntiles, pblk, e_full, wt, l):
        """J^T J, J^T e of ordered subset l with the reference's pairing (orc_normal_eq_os): e_full is
        the chunk's residual as the LM holds it (weighted by wt), wt its sqrt-weights or None"""
        n8 = 8 * self.pr.N
        JTJ = np.zeros((n8, n8))
        JTe = np.zeros(n8)
        pblk = np.ascontiguousarray(pblk, dtype=np.float64)
        e_full = np.ascontiguousarray(e_full, dtype=np.float64)
        wt = None if wt is None else np.ascontiguousarray(wt, dtype=np.float64)
        self.L.orc_normal_eq_os(C.byref(self.P), k, t0, ntiles, _d(pblk), _d(e_full),
                                _d(wt) if wt is not None else None, l, _d(JTJ.reshape(-1)), _d(JTe))
        return JTJ, JTe

    def lm_chunk(self, k, t0, ntiles, pblk, xd, itmax, opts=(1e-3, 1e-15, 1e-15, 1e-20, -1e-6),
                 linsolv=0, os_=False):
        p = np.ascontiguousarray(pblk, dtype=np.float64).copy()
        info = np.zeros(10)
        o = np.array(opts)
        xd = np.ascontiguousarray(xd)
        self.L.orc_lm_chunk(C.byref(self.P), k, t0, ntiles, _d(p), _d(xd), itmax, _d(o), linsolv,
                            int(os_), _d(info))
        return p, info

    def rlm_chunk(self, k, t0, ntiles, pblk, xd, itmax, linsolv=0, os_=False, nulow=2.0,
                  nuhigh=30.0, nu0=2.0):
        p = np.ascontiguousarray(pblk, dtype=np.float64).copy()
        info = np.zeros(10)
        nu = C.c_double(nu0)
        xd = np.ascontiguousarray(xd)
        self.L.orc_rlm_chunk(C.byref(self.P), k, t0, ntiles, _d(p), _d(xd), itmax, linsolv,
                             int(os_), nulow, nuhigh, C.byref(nu), _d(info))
        return p, info, nu.value

    def rtr_chunk(self, k, t0, ntiles, pblk, xd, kind, itmax_a, itmax_b, nulow=2.0, nuhigh=30.0,
                  nu0=2.0, nu_joined=True, tensor=False, Y=None, BZ=None, rho=0.0):
        """RTR (kind 4), robust RTR (5), NSD (6) of one chunk on hidden data xd.  tensor: with the
        per-baseline tensor arithmetic of the product's kernels instead of the per-row evaluators"""
        p = np.ascontiguousarray(pblk, dtype=np.float64).copy()
        info = np.zeros(10)
        nu = C.c_double(nu0)
        xd = np.ascontiguousarray(xd)
        if Y is not None:  # consensus terms of this block (rtr_solve_nocuda_robust_admm)
            Y = np.ascontiguousarray(Y, dtype=np.float64)
            BZ = np.ascontiguousarray(BZ, dtype=np.float64)
        yp, zp = (_d(Y), _d(BZ)) if Y is not None else (None, None)
        if tensor:
            self.HT.harness_rtr_solve_tensor(C.byref(self.P), k, t0, ntiles, _d(xd), kind, _d(p),
                                             itmax_a, itmax_b, nulow, nuhigh, C.byref(nu),
                                             _d(info), int(nu_joined), yp, zp, rho)
            return p, info, nu.value
        self.H.harness_rtr_solve_admm(C.byref(self.P), self.pr.N, self.pr.Nbase, k, t0, ntiles,
                                      _d(xd), kind, _d(p), itmax_a, itmax_b, nulow, nuhigh,
                                      C.byref(nu), _d(info), int(nu_joined), yp, zp, rho)
        return p, info, nu.value

    # ---- the per-row RTR evaluators (orc_rtr_*) on hidden data y of tiles [t0, t0 + ntiles) ----
    def rtr_raw(self, k, t0, ntiles, y, x, eta=None, wt=None, vec=True):
        """(cost, raw station sums [8N] or None): gradient sums (eta None) or Hessian terms"""
        y = np.ascontiguousarray(y, dtype=np.float64)
        x = np.ascontiguousarray(x, dtype=np.float64)
        v = np.zeros(8 * self.pr.N) if vec else None
        e = None if eta is None else np.ascontiguousarray(eta, dtype=np.float64)
        w = None if wt is None else np.ascontiguousarray(wt, dtype=np.float64)
        c = self.L.orc_rtr_raw(C.byref(self.P), k, t0, ntiles, _d(y), _d(w) if w is not None else None,
                               _d(x), _d(e) if e is not None else None, _d(v) if vec else None)
        return c, v

    def rtr_counts(self, t0, ntiles):
        c = np.zeros(self.pr.N)
        self.L.orc_rtr_counts(C.byref(self.P), t0, ntiles, _d(c))
        return c

    def rtr_weights(self, k, t0, ntiles, y, x, nu):
        """(sum(log w - w) over unflagged rows / all rows, row weights; flagged rows 0)"""
        y = np.ascontiguousarray(y, dtype=np.float64)
        x = np.ascontiguousarray(x, dtype=np.float64)
        wt = np.zeros(ntiles * self.pr.Nbase)
        s = self.L.orc_rtr_weights(C.byref(self.P), k, t0, ntiles, _d(y), _d(x), nu, _d(wt))
        return s, wt

    def update_w_and_nu(self, nu0, ed, nulow=2.0, nuhigh=30.0):
        w = np.zeros(len(ed))
        nu = self.L.orc_update_w_and_nu(nu0, _d(w), _d(np.ascontiguousarray(ed)), len(ed), nulow,
                                        nuhigh)
        return nu, w

    def sagefit(self, x, pp, max_emiter=3, max_iter=2, max_lbfgs=10, lbfgs_m=7, linsolv=0,
                solver_mode=1, nulow=2.0, nuhigh=30.0, **_ignored):
        nu, r0, r1 = C.c_double(0), C.c_double(0), C.c_double(0)
        rv = self.L.orc_sagefit(C.byref(self.P), _d(x), _d(pp), max_emiter, max_iter, max_lbfgs,
                                lbfgs_m, linsolv, solver_mode, nulow, nuhigh, C.byref(nu),
                                C.byref(r0), C.byref(r1))
        return rv, nu.value, r0.value, r1.value

    def lbfgs_trace(self, x, pp, itmax, M, robust=False, nu=2.0):
        """orc_lbfgs with its trace.  returns dict(p [final], niter, alphak, ncost, slot, gnorm
        [per iteration], iterates [niter, m], margin [smallest line-search decision margin])"""
        p = np.array(pp, dtype=np.float64)
        n = max(itmax, 1)
        alphak, gnorm = np.zeros(n), np.zeros(n)
        ncost = np.zeros(n, dtype=np.int64)
        slot = np.zeros(n, dtype=np.int32)
        it = np.zeros((n, self.m))
        tr = orc_lbfgs_trace(_d(alphak), ncost.ctypes.data_as(C.POINTER(C.c_longlong)),
                             slot.ctypes.data_as(ip), _d(gnorm), _d(it.reshape(-1)), 0, 0.0)
        self.L.orc_lbfgs_traced(C.byref(self.P), _d(p), _d(np.ascontiguousarray(x)), itmax, M,
                                int(robust), nu, C.byref(tr))
        k = tr.niter
        return dict(p=p, niter=k, alphak=alphak[:k], ncost=ncost[:k], slot=slot[:k],
                    gnorm=gnorm[:k], iterates=it[:k], margin=tr.margin)

    def bfgsfit(self, x, pp, max_lbfgs=10, lbfgs_m=7, solver_mode=1, mean_nu=2.0, **_ignored):
        r0, r1 = C.c_double(0), C.c_double(0)
        rv = self.L.orc_bfgsfit(C.byref(self.P), _d(x), _d(pp), max_lbfgs, lbfgs_m, solver_mode,
                                mean_nu, C.byref(r0), C.byref(r1))
        return rv, r0.value, r1.value


class OracleSky:
    def __init__(self, clusters):
        L = C.CDLL(ORC_PATH)
        self.L = L
        ps = C.POINTER(orc_sky)
        d, i = C.c_double, C.c_int
        L.orc_coherencies.argtypes = [ps, dp, dp, dp, i, d, d, d, d, up, dp]
        L.orc_predict_multifreq.argtypes = [ps, dp, dp, dp, i, dp, i, d, i, dp]
        cat = lambda name, default=None: np.ascontiguousarray(np.concatenate(
            [np.asarray(cl.get(name, default(cl) if default else None), dtype=np.float64)
             for cl in clusters]))
        K = [len(cl["ll"]) for cl in clusters]
        self.src0 = np.concatenate([[0], np.cumsum(K)]).astype(np.int32)
        self.a = {}
        for n in ("ll", "mm", "nn", "sI", "sQ", "sU", "sV"):
            self.a[n] = cat(n)
        self.a["sI0"] = cat("sI0", lambda cl: cl["sI"])
        self.a["sQ0"] = cat("sQ0", lambda cl: cl["sQ"])
        self.a["sU0"] = cat("sU0", lambda cl: cl["sU"])
        self.a["sV0"] = cat("sV0", lambda cl: cl["sV"])
        self.a["f0"] = cat("f0", lambda cl: np.full(len(cl["ll"]), 150e6))
        for n in ("spec_idx", "spec_idx1", "spec_idx2"):
            self.a[n] = cat(n, lambda cl: np.zeros(len(cl["ll"])))
        self.stype = np.ascontiguousarray(np.concatenate(
            [np.asarray(cl.get("stype", np.zeros(len(cl["ll"]))), dtype=np.uint8) for cl in clusters]))
        self.gauss = np.ascontiguousarray(np.concatenate(
            [np.asarray(cl.get("gauss", np.zeros((len(cl["ll"]), 8))), dtype=np.float64)
             for cl in clusters]).reshape(-1))
        S = orc_sky()
        S.M = len(clusters)
        S.src0 = self.src0.ctypes.data_as(ip)
        for n, arr in self.a.items():
            setattr(S, n, _d(arr))
        S.stype = self.stype.ctypes.data_as(up)
        S.gauss = _d(self.gauss)
        self.S = S

    def coherencies(self, u, v, w, freq0, fdelta, uvmin=0.0, uvmax=1e9, flag=None):
        nrow = len(u)
        coh = np.zeros(4 * self.S.M * nrow, dtype=np.complex128)
        self.L.orc_coherencies(C.byref(self.S), _d(u), _d(v), _d(w), nrow, freq0, fdelta, uvmin,
                               uvmax, flag.ctypes.data_as(up) if flag is not None else None,
                               coh.view(np.float64).ctypes.data_as(dp))
        return coh

    def predict_multifreq(self, u, v, w, freqs, fdelta, add_to_data, x):
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        self.L.orc_predict_multifreq(C.byref(self.S), _d(u), _d(v), _d(w), len(u), _d(freqs),
                                     len(freqs), fdelta, add_to_data, _d(x))
        return x
