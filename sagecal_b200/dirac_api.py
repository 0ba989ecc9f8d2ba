"""ctypes view of the Dirac C API for the direction-dependent calibration hot path.

The structs and prototypes below are the *interface* the reference driver (`sagecal_gpu`,
src/MS/fullbatch_mode.cpp:371-446) binds against; they are restated from
src/lib/Dirac/Dirac_common.h:173-195 (clus_source_t, baseline_t), Dirac.h:1651,1683
(sagefit_visibilities, bfgsfit_visibilities) and src/lib/Radio/Dirac_radio.h:209,659
(precalculate_coherencies, predict_visibilities_multifreq).

`DiracAPI(path)` binds any shared library that implements this ABI.  The product library is
`sagecal_b200/libdirac_b200.so` (see `sagecal_b200.lib`); the test suite additionally binds the
compiled reference through the very same class, which is what makes the parity tests read like
"call both, compare".  Nothing in this package loads that library.
"""
from __future__ import annotations

import ctypes as C
import numpy as np

c_double_p = C.POINTER(C.c_double)
c_int_p = C.POINTER(C.c_int)
c_ubyte_p = C.POINTER(C.c_ubyte)

STYPE_POINT = 0
STYPE_GAUSSIAN = 1
STYPE_DISK = 2
STYPE_RING = 3
STYPE_SHAPELET = 4

# solver_mode values, Dirac.h:1607-1613
SM_OSLM_LBFGS = 0
SM_LM_LBFGS = 1
SM_RLM_RLBFGS = 2
SM_OSLM_OSRLM_RLBFGS = 3
SM_RTR_OSLM_LBFGS = 4
SM_RTR_OSRLM_RLBFGS = 5
SM_NSD_RLBFGS = 6


class baseline_t(C.Structure):
    """Dirac_common.h:190-195 — row -> (sta1, sta2, flag)."""
    _fields_ = [("sta1", C.c_int), ("sta2", C.c_int), ("flag", C.c_ubyte)]


class clus_source_t(C.Structure):
    """Dirac_common.h:173-187 — one cluster (direction) of the sky model."""
    _fields_ = [
        ("N", C.c_int), ("id", C.c_int),
        ("ll", c_double_p), ("mm", c_double_p), ("nn", c_double_p),
        ("sI", c_double_p), ("sQ", c_double_p), ("sU", c_double_p), ("sV", c_double_p),
        ("ra", c_double_p), ("dec", c_double_p),
        ("stype", c_ubyte_p), ("ex", C.POINTER(C.c_void_p)),
        ("nchunk", C.c_int), ("p", c_int_p),
        ("sI0", c_double_p), ("sQ0", c_double_p), ("sU0", c_double_p), ("sV0", c_double_p),
        ("f0", c_double_p), ("spec_idx", c_double_p), ("spec_idx1", c_double_p),
        ("spec_idx2", c_double_p),
    ]


class persistent_data_t(C.Structure):
    """include/dirac_b200.h: the prefix of the reference's struct this library uses"""
    _fields_ = [("y", C.c_void_p), ("s", C.c_void_p), ("rho", C.c_void_p), ("nfilled", C.c_int),
                ("vacant", C.c_int), ("lbfgs_m", C.c_int), ("m", C.c_int), ("Nt", C.c_int)]


class exinfo_gaussian(C.Structure):
    """Dirac_radio.h exinfo_gaussian — extended (Gaussian) source shape."""
    _fields_ = [("eX", C.c_double), ("eY", C.c_double), ("eP", C.c_double),
                ("cxi", C.c_double), ("sxi", C.c_double), ("cphi", C.c_double),
                ("sphi", C.c_double), ("use_projection", C.c_int)]


class exinfo_disk(C.Structure):
    """Dirac_common.h exinfo_disk / exinfo_ring (same layout)."""
    _fields_ = [("eX", C.c_double), ("cxi", C.c_double), ("sxi", C.c_double),
                ("cphi", C.c_double), ("sphi", C.c_double), ("use_projection", C.c_int)]


class exinfo_shapelet(C.Structure):
    """Dirac_common.h exinfo_shapelet — n0 x n0 shapelet modes."""
    _fields_ = [("n0", C.c_int), ("beta", C.c_double), ("modes", C.POINTER(C.c_double)),
                ("eX", C.c_double), ("eY", C.c_double), ("eP", C.c_double),
                ("cxi", C.c_double), ("sxi", C.c_double), ("cphi", C.c_double),
                ("sphi", C.c_double), ("use_projection", C.c_int)]


assert C.sizeof(baseline_t) == 12


def dptr(a: np.ndarray):
    assert a.dtype == np.float64 and a.flags.c_contiguous
    return a.ctypes.data_as(c_double_p)


def cptr(a: np.ndarray):
    """complex128 array viewed as the `complex double *` the API expects."""
    assert a.dtype == np.complex128 and a.flags.c_contiguous
    return a.ctypes.data_as(c_double_p)


class SkyModel:
    """Owns the numpy buffers behind an array of clus_source_t."""

    def __init__(self, clusters, N, keep_alive=None, p_base=0):
        """clusters: list of dict(ll,mm,nn,sI,sQ,sU,sV[,stype,nchunk,f0,spec_idx...,gauss]).
        p_base: offset of the first cluster's Jones block in the parameter vector (a shard of a
        larger sky model keeps the global offsets)."""
        self.M = len(clusters)
        self.arr = (clus_source_t * self.M)()
        self._keep = []
        off = int(p_base)
        self.nchunk = []
        for k, cl in enumerate(clusters):
            K = len(cl["ll"])
            cs = self.arr[k]
            cs.N = K
            cs.id = int(cl.get("id", k))
            for name in ("ll", "mm", "nn", "sI", "sQ", "sU", "sV"):
                a = np.ascontiguousarray(cl[name], dtype=np.float64)
                self._keep.append(a)
                setattr(cs, name, dptr(a))
            for name in ("ra", "dec"):
                a = np.ascontiguousarray(cl.get(name, np.zeros(K)), dtype=np.float64)
                self._keep.append(a)
                setattr(cs, name, dptr(a))
            st = np.ascontiguousarray(cl.get("stype", np.zeros(K)), dtype=np.uint8)
            self._keep.append(st)
            cs.stype = st.ctypes.data_as(c_ubyte_p)
            ex = (C.c_void_p * K)()
            gauss = cl.get("gauss")
            if gauss is not None:
                for s in range(K):
                    if st[s] == STYPE_GAUSSIAN:
                        g = exinfo_gaussian(*[float(v) for v in gauss[s][:7]], int(gauss[s][7]))
                        self._keep.append(g)
                        ex[s] = C.cast(C.pointer(g), C.c_void_p)
            # disks / rings: cl["disk"][s] = (eX, cxi, sxi, cphi, sphi, use_projection);
            # shapelets: cl["shapelet"][s] = dict(n0, beta, modes, eX, eY, eP[, cxi, sxi, cphi, sphi,
            # use_projection])
            for s_, g_ in (cl.get("disk") or {}).items():
                g = exinfo_disk(*[float(v) for v in g_[:5]], int(g_[5]))
                self._keep.append(g)
                ex[s_] = C.cast(C.pointer(g), C.c_void_p)
            for s_, g_ in (cl.get("shapelet") or {}).items():
                modes = np.ascontiguousarray(g_["modes"], dtype=np.float64)
                assert modes.size == g_["n0"] ** 2
                g = exinfo_shapelet(int(g_["n0"]), float(g_["beta"]), dptr(modes), float(g_["eX"]),
                                    float(g_["eY"]), float(g_["eP"]), float(g_.get("cxi", 1.0)),
                                    float(g_.get("sxi", 0.0)), float(g_.get("cphi", 1.0)),
                                    float(g_.get("sphi", 0.0)), int(g_.get("use_projection", 0)))
                self._keep.extend([modes, g])
                ex[s_] = C.cast(C.pointer(g), C.c_void_p)
            self._keep.append(ex)
            cs.ex = C.cast(ex, C.POINTER(C.c_void_p))
            nchunk = int(cl.get("nchunk", 1))
            cs.nchunk = nchunk
            self.nchunk.append(nchunk)
            p = np.array([off + c * 8 * N for c in range(nchunk)], dtype=np.int32)
            off += nchunk * 8 * N
            self._keep.append(p)
            cs.p = p.ctypes.data_as(c_int_p)
            # multi-channel spectral model (residual.c:1177-1210); default: flat spectrum
            for name, src in (("sI0", "sI"), ("sQ0", "sQ"), ("sU0", "sU"), ("sV0", "sV")):
                a = np.ascontiguousarray(cl.get(name, cl[src]), dtype=np.float64)
                self._keep.append(a)
                setattr(cs, name, dptr(a))
            f0 = np.ascontiguousarray(cl.get("f0", np.full(K, 150e6)), dtype=np.float64)
            self._keep.append(f0)
            cs.f0 = dptr(f0)
            for name in ("spec_idx", "spec_idx1", "spec_idx2"):
                a = np.ascontiguousarray(cl.get(name, np.zeros(K)), dtype=np.float64)
                self._keep.append(a)
                setattr(cs, name, dptr(a))
        self.Mt = sum(self.nchunk)
        self.nparam = off - int(p_base)


class elementcoeff(C.Structure):
    """Dirac_common.h:153-162 — element beam coefficient tables (filled by the REFERENCE library's
    set_elementcoeffs / set_elementcoeffs_wb; this library only evaluates them)"""
    _fields_ = [("M", C.c_int), ("Nmodes", C.c_int), ("Nf", C.c_int), ("beta", C.c_double),
                ("pattern_phi", C.c_void_p), ("pattern_theta", C.c_void_p),
                ("preamble", C.c_void_p)]


class BeamSetup:
    """the beam arguments of the *_withbeam calls, with the numpy buffers behind them"""

    def __init__(self, bf_type, b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0, longitude, latitude,
                 time_utc, elem_xyz, ecoeff, doBeam, Nelem=None):
        """elem_xyz: per station an array [n][3] of element positions (STAT_TILE: the 16 dipoles of a
        tile first, then the tile centroids; Nelem then counts the tiles)"""
        self.bf_type, self.doBeam = int(bf_type), int(doBeam)
        self.s = [C.c_double(float(v)) for v in (b_ra0, b_dec0, ph_ra0, ph_dec0, ph_freq0)]
        self.lon = np.ascontiguousarray(longitude, dtype=np.float64)
        self.lat = np.ascontiguousarray(latitude, dtype=np.float64)
        self.t = np.ascontiguousarray(time_utc, dtype=np.float64)
        self.tilesz = len(self.t)
        N = len(self.lon)
        self.xyz = [np.ascontiguousarray(np.asarray(e, dtype=np.float64).T) for e in elem_xyz]
        extra = 16 if self.bf_type == 2 else 0
        self.Nelem = np.ascontiguousarray(
            Nelem if Nelem is not None else [e.shape[1] - extra for e in self.xyz], dtype=np.int32)
        mk = lambda axis: (c_double_p * N)(*[dptr(e[axis]) for e in self.xyz])
        self.xx, self.yy, self.zz = mk(0), mk(1), mk(2)
        self.ecoeff = ecoeff

    def head(self):
        return (self.bf_type, *self.s, dptr(self.lon), dptr(self.lat), dptr(self.t))

    def tail(self):
        ec = C.byref(self.ecoeff) if self.ecoeff is not None else None
        return (self.Nelem.ctypes.data_as(c_int_p), self.xx, self.yy, self.zz, ec, self.doBeam)


def make_barr(sta1, sta2, flag):
    n = len(sta1)
    barr = (baseline_t * n)()
    view = np.ctypeslib.as_array(C.cast(barr, C.POINTER(C.c_int)), shape=(n, 3))
    view[:, 0] = sta1
    view[:, 1] = sta2
    view[:, 2] = 0
    fl = np.ctypeslib.as_array(C.cast(barr, c_ubyte_p), shape=(n, 12))
    fl[:, 8] = np.asarray(flag, dtype=np.uint8)
    return barr


def _ignorelist(ignorelist, M):
    """the int[M] ignore list of the simulation calls; None: no cluster ignored"""
    ign = np.zeros(M, dtype=np.int32) if ignorelist is None else np.asarray(ignorelist, dtype=np.int32)
    assert ign.shape == (M,)
    return np.ascontiguousarray(ign)


def barr_to_numpy(barr, n):
    view = np.ctypeslib.as_array(C.cast(barr, C.POINTER(C.c_int)), shape=(n, 3))
    fl = np.ctypeslib.as_array(C.cast(barr, c_ubyte_p), shape=(n, 12))
    return view[:, 0].copy(), view[:, 1].copy(), fl[:, 8].copy()


class DiracAPI:
    """Binds the hot-path entry points of a Dirac-ABI shared library."""

    def __init__(self, path: str, lib=None):
        self.path = path
        self.lib = lib if lib is not None else C.CDLL(path, mode=C.RTLD_GLOBAL)
        L = self.lib
        bp = C.POINTER(baseline_t)
        cp = C.POINTER(clus_source_t)
        d = C.c_double
        i = C.c_int
        dp = c_double_p

        L.sagefit_visibilities.restype = i
        L.sagefit_visibilities.argtypes = [dp, dp, dp, dp, i, i, i, bp, cp, dp, i, i, d, d, dp, d,
                                           i, i, i, i, i, i, i, i, d, d, i, dp, dp, dp]
        L.bfgsfit_visibilities.restype = i
        L.bfgsfit_visibilities.argtypes = [dp, dp, dp, dp, i, i, i, bp, cp, dp, i, i, d, d, dp, d,
                                           i, i, i, i, i, d, dp, dp]
        L.precalculate_coherencies.restype = i
        L.precalculate_coherencies.argtypes = [dp, dp, dp, dp, i, i, bp, cp, i, d, d, d, d, d, d, i]
        L.predict_visibilities_multifreq.restype = i
        L.predict_visibilities_multifreq.argtypes = [dp, dp, dp, dp, i, i, i, bp, cp, i, dp, i,
                                                     d, d, d, i, i]
        L.calculate_residuals_multifreq.restype = i
        L.calculate_residuals_multifreq.argtypes = [dp, dp, dp, dp, dp, i, i, i, bp, cp, i, dp, i,
                                                    d, d, d, i, i, d, i]
        L.predict_visibilities_multifreq_withsol.restype = i
        L.predict_visibilities_multifreq_withsol.argtypes = [dp, dp, dp, dp, dp, c_int_p, i, i, i, bp,
                                                             cp, i, dp, i, d, d, d, i, i, i, d, i]
        L.generate_baselines.restype = i
        L.generate_baselines.argtypes = [i, i, i, bp, i]
        L.preset_flags_and_data.restype = i
        L.preset_flags_and_data.argtypes = [i, dp, bp, dp, i]
        if hasattr(L, "whiten_data"):
            L.whiten_data.restype = None
            L.whiten_data.argtypes = [i, dp, dp, dp, d, i]
        if hasattr(L, "calculate_residuals_multifreq"):
            L.calculate_residuals_multifreq.restype = i
            L.calculate_residuals_multifreq.argtypes = [dp, dp, dp, dp, dp, i, i, i, bp, cp, i, dp,
                                                        i, d, d, d, i, i, d, i]

    # -- thin pythonic wrappers (argument order and meaning exactly as the C API) -----------------
    def generate_baselines(self, Nbase, tilesz, N, Nt=4):
        barr = (baseline_t * (Nbase * tilesz))()
        self.lib.generate_baselines(Nbase, tilesz, N, barr, Nt)
        return barr

    def preset_flags_and_data(self, flag, barr, x, Nt=4):
        return self.lib.preset_flags_and_data(len(flag), dptr(flag), barr, dptr(x), Nt)

    def whiten_data(self, x, u, v, freq0, Nt=4):
        """uv taper of the data in place (Dirac.h:841); u, v in seconds as everywhere in the API"""
        self.lib.whiten_data(len(u), dptr(x), dptr(u), dptr(v), freq0, Nt)

    def precalculate_coherencies(self, u, v, w, N, Nbase1, barr, sky: SkyModel, freq0, fdelta,
                                 tdelta=10.0, dec0=1.0, uvmin=0.0, uvmax=1e9, Nt=4):
        coh = np.zeros(4 * sky.M * Nbase1, dtype=np.complex128)
        self.lib.precalculate_coherencies(dptr(u), dptr(v), dptr(w), cptr(coh), N, Nbase1, barr,
                                          sky.arr, sky.M, freq0, fdelta, tdelta, dec0, uvmin,
                                          uvmax, Nt)
        return coh

    def predict_visibilities_multifreq(self, u, v, w, x, N, Nbase, tilesz, barr, sky: SkyModel,
                                       freqs, fdelta, tdelta=10.0, dec0=1.0, Nt=4, add_to_data=1):
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        return self.lib.predict_visibilities_multifreq(
            dptr(u), dptr(v), dptr(w), dptr(x), N, Nbase, tilesz, barr, sky.arr, sky.M,
            dptr(freqs), len(freqs), fdelta, tdelta, dec0, Nt, add_to_data)

    def calculate_residuals_multifreq(self, u, v, w, p, x, N, Nbase, tilesz, barr, sky: SkyModel,
                                      freqs, fdelta, tdelta=10.0, dec0=1.0, Nt=4, ccid=-99999,
                                      rho=1e-9, phase_only=0):
        """x[chan][row][8]: data in, residual (optionally corrected by cluster `ccid`) out"""
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        return self.lib.calculate_residuals_multifreq(
            dptr(u), dptr(v), dptr(w), dptr(p), dptr(x), N, Nbase, tilesz, barr, sky.arr, sky.M,
            dptr(freqs), len(freqs), fdelta, tdelta, dec0, Nt, ccid, rho, phase_only)

    def predict_visibilities_multifreq_withsol(self, u, v, w, p, x, N, Nbase, tilesz, barr,
                                               sky: SkyModel, freqs, fdelta, ignorelist=None,
                                               tdelta=10.0, dec0=1.0, Nt=4, add_to_data=1,
                                               ccid=-99999, rho=1e-9, phase_only=0):
        """simulation with solutions (Dirac_radio.h:666).  x[chan][row][8] in/out; ignorelist: one
        flag per cluster position, nonzero skips the cluster (None: predict every cluster);
        add_to_data 1 model only, 2 add, 3 subtract; then the optional correction by cluster ccid"""
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        ign = _ignorelist(ignorelist, sky.M)
        return self.lib.predict_visibilities_multifreq_withsol(
            dptr(u), dptr(v), dptr(w), dptr(p), dptr(x), ign.ctypes.data_as(c_int_p), N, Nbase,
            tilesz, barr, sky.arr, sky.M, dptr(freqs), len(freqs), fdelta, tdelta, dec0, Nt,
            add_to_data, ccid, rho, phase_only)

    def calculate_residuals(self, u, v, w, p, x, N, Nbase, tilesz, barr, sky: SkyModel, freq0, fdelta,
                            tdelta=10.0, dec0=1.0, Nt=4, ccid=-99999, rho=1e-9):
        """single-channel residual (Dirac_radio.h:639).  x[row][8]: data in, residual (optionally
        corrected by cluster `ccid`) out"""
        L = self.lib
        L.calculate_residuals.restype = C.c_int
        L.calculate_residuals.argtypes = [c_double_p] * 5 + [C.c_int] * 3 + [
            C.POINTER(baseline_t), C.POINTER(clus_source_t), C.c_int] + [C.c_double] * 4 + [
            C.c_int, C.c_int, C.c_double]
        return L.calculate_residuals(dptr(u), dptr(v), dptr(w), dptr(p), dptr(x), N, Nbase, tilesz,
                                     barr, sky.arr, sky.M, freq0, fdelta, tdelta, dec0, Nt, ccid, rho)

    def bfgsfit_channels(self, u, v, w, xo, N, Nbase, tilesz, barr, sky: SkyModel, freqs, deltafch, p,
                         uvmin=0.0, uvmax=1e9, max_lbfgs=10, lbfgs_m=7, solver_mode=SM_LM_LBFGS,
                         mean_nu=2.0, ccid=-99999, rho=1e-9, keep_pfreq=True):
        """dirac_b200_bfgsfit_channels: the per-channel refinement of one interval on a resident
        problem.  xo [Nchan][row][8] data -> residual, p start Jones -> last channel's solution,
        barr flags updated by the uv cut of every channel.
        returns (retval, res_00 [Nchan], res_01 [Nchan], pfreq [Nchan, 8 N Mt] or None)"""
        L = self.lib
        L.dirac_b200_bfgsfit_channels.restype = C.c_int
        L.dirac_b200_bfgsfit_channels.argtypes = [c_double_p] * 4 + [C.c_int] * 3 + [
            C.POINTER(baseline_t), C.POINTER(clus_source_t), C.c_int, C.c_int, c_double_p, C.c_int,
            C.c_double, C.c_double, C.c_double, c_double_p, C.c_int, C.c_int, C.c_int, C.c_double,
            C.c_int, C.c_double, c_double_p, c_double_p, c_double_p]
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        nchan = len(freqs)
        r0, r1 = np.zeros(nchan), np.zeros(nchan)
        pfreq = np.zeros((nchan, len(p))) if keep_pfreq else None
        rv = L.dirac_b200_bfgsfit_channels(
            dptr(u), dptr(v), dptr(w), dptr(xo), N, Nbase, tilesz, barr, sky.arr, sky.M, sky.Mt,
            dptr(freqs), nchan, deltafch, uvmin, uvmax, dptr(p), max_lbfgs, lbfgs_m, solver_mode,
            mean_nu, ccid, rho, dptr(r0), dptr(r1),
            dptr(pfreq.reshape(-1)) if keep_pfreq else None)
        return rv, r0, r1, pfreq

    def recalculate_diffuse_coherencies(self, u, v, w, x, N, barr, sky: SkyModel, freq0, fdelta, cid,
                                        sh_n0, sh_beta, Z, tdelta=10.0, dec0=1.0, uvmin=0.0,
                                        uvmax=1e9, Nt=4, use_cuda=0):
        """coherencies of cluster cid rewritten from the spatial model Z (Dirac_radio.h:228).
        x: [row][M][4] complex, in/out (only cluster cid changes); Z: 2N x 2G complex (G = sh_n0^2),
        passed column major"""
        L = self.lib
        L.recalculate_diffuse_coherencies.restype = C.c_int
        L.recalculate_diffuse_coherencies.argtypes = [
            c_double_p, c_double_p, c_double_p, c_double_p, C.c_int, C.c_int, C.POINTER(baseline_t),
            C.POINTER(clus_source_t), C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
            C.c_double, C.c_double, C.c_int, C.c_int, C.c_double, c_double_p, C.c_int, C.c_int]
        Zf = np.asfortranarray(Z, dtype=np.complex128).reshape(-1, order="F")
        return L.recalculate_diffuse_coherencies(
            dptr(u), dptr(v), dptr(w), cptr(x), N, len(u), barr, sky.arr, sky.M, freq0, fdelta,
            tdelta, dec0, uvmin, uvmax, cid, sh_n0, sh_beta, cptr(Zf), Nt, use_cuda)

    # ---- station beams (Dirac_radio.h:472-490) ----
    def precalculate_coherencies_withbeam(self, u, v, w, N, Nbase1, barr, sky, freq0, fdelta, beam,
                                          tdelta=10.0, dec0=1.0, uvmin=0.0, uvmax=1e9, Nt=4):
        coh = np.zeros(4 * sky.M * Nbase1, dtype=np.complex128)
        self.lib.precalculate_coherencies_withbeam(
            dptr(u), dptr(v), dptr(w), cptr(coh), N, Nbase1, barr, sky.arr, sky.M,
            C.c_double(freq0), C.c_double(fdelta), C.c_double(tdelta), C.c_double(dec0),
            C.c_double(uvmin), C.c_double(uvmax), *beam.head(), beam.tilesz, *beam.tail(), Nt)
        return coh

    def precalculate_coherencies_multifreq(self, u, v, w, N, Nbase1, barr, sky, freqs, fdelta,
                                           beam=None, tdelta=10.0, dec0=1.0, uvmin=0.0, uvmax=1e9,
                                           Nt=4):
        """coh[chan][row][cluster][4] (predict.c:745); beam: the _withbeam variant"""
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        coh = np.zeros(4 * sky.M * Nbase1 * len(freqs), dtype=np.complex128)
        head = (dptr(u), dptr(v), dptr(w), cptr(coh), N, Nbase1, barr, sky.arr, sky.M, dptr(freqs),
                len(freqs), C.c_double(fdelta), C.c_double(tdelta), C.c_double(dec0),
                C.c_double(uvmin), C.c_double(uvmax))
        if beam is None:
            self.lib.precalculate_coherencies_multifreq(*head, Nt)
        else:
            self.lib.precalculate_coherencies_multifreq_withbeam(*head, *beam.head(), beam.tilesz,
                                                                 *beam.tail(), Nt)
        return coh

    def predict_visibilities_multifreq_withbeam(self, u, v, w, x, N, Nbase, tilesz, barr, sky, freqs,
                                                fdelta, beam, tdelta=10.0, dec0=1.0, Nt=4,
                                                add_to_data=1):
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        return self.lib.predict_visibilities_multifreq_withbeam(
            dptr(u), dptr(v), dptr(w), dptr(x), N, Nbase, tilesz, barr, sky.arr, sky.M, dptr(freqs),
            len(freqs), C.c_double(fdelta), C.c_double(tdelta), C.c_double(dec0), *beam.head(),
            *beam.tail(), Nt, add_to_data)

    def calculate_residuals_multifreq_withbeam(self, u, v, w, p, x, N, Nbase, tilesz, barr, sky,
                                               freqs, fdelta, beam, tdelta=10.0, dec0=1.0, Nt=4,
                                               ccid=-99999, rho=1e-9, phase_only=0):
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        return self.lib.calculate_residuals_multifreq_withbeam(
            dptr(u), dptr(v), dptr(w), dptr(p), dptr(x), N, Nbase, tilesz, barr, sky.arr, sky.M,
            dptr(freqs), len(freqs), C.c_double(fdelta), C.c_double(tdelta), C.c_double(dec0),
            *beam.head(), *beam.tail(), Nt, ccid, C.c_double(rho), phase_only)

    def predict_visibilities_multifreq_withsol_withbeam(self, u, v, w, p, x, N, Nbase, tilesz, barr,
                                                        sky, freqs, fdelta, beam, ignorelist=None,
                                                        tdelta=10.0, dec0=1.0, Nt=4, add_to_data=1,
                                                        ccid=-99999, rho=1e-9, phase_only=0,
                                                        gpu_twin=False):
        """predict_visibilities_multifreq_withsol with station beams (Dirac_radio.h:490);
        gpu_twin: through its GPU-build name predict_visibilities_withsol_withbeam_gpu (:529)"""
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        ign = _ignorelist(ignorelist, sky.M)
        fn = (self.lib.predict_visibilities_withsol_withbeam_gpu if gpu_twin
              else self.lib.predict_visibilities_multifreq_withsol_withbeam)
        return fn(dptr(u), dptr(v), dptr(w), dptr(p), dptr(x), ign.ctypes.data_as(c_int_p), N, Nbase,
                  tilesz, barr, sky.arr, sky.M, dptr(freqs), len(freqs), C.c_double(fdelta),
                  C.c_double(tdelta), C.c_double(dec0), *beam.head(), *beam.tail(), Nt, add_to_data,
                  ccid, C.c_double(rho), phase_only)

    def sagefit_visibilities(self, u, v, w, x, N, Nbase, tilesz, barr, sky: SkyModel, coh, pp,
                             freq0=150e6, fdelta=195.3e3, uvmin=0.0, Nt=4, max_emiter=3,
                             max_iter=2, max_lbfgs=10, lbfgs_m=7, gpu_threads=128, linsolv=0,
                             solver_mode=SM_LM_LBFGS, nulow=2.0, nuhigh=30.0, randomize=0):
        """x (data -> residual) and pp (Jones) are updated in place; returns
        (retval, mean_nu, res_0, res_1)."""
        mean_nu = C.c_double(0.0)
        res0 = C.c_double(0.0)
        res1 = C.c_double(0.0)
        rv = self.lib.sagefit_visibilities(
            dptr(u), dptr(v), dptr(w), dptr(x), N, Nbase, tilesz, barr, sky.arr, cptr(coh),
            sky.M, sky.Mt, freq0, fdelta, dptr(pp), uvmin, Nt, max_emiter, max_iter, max_lbfgs,
            lbfgs_m, gpu_threads, linsolv, solver_mode, nulow, nuhigh, randomize,
            C.byref(mean_nu), C.byref(res0), C.byref(res1))
        return rv, mean_nu.value, res0.value, res1.value

    def bfgsfit_visibilities(self, u, v, w, x, N, Nbase, tilesz, barr, sky: SkyModel, coh, pp,
                             freq0=150e6, fdelta=195.3e3, uvmin=0.0, Nt=4, max_lbfgs=10,
                             lbfgs_m=7, gpu_threads=128, solver_mode=SM_LM_LBFGS, mean_nu=2.0):
        res0 = C.c_double(0.0)
        res1 = C.c_double(0.0)
        rv = self.lib.bfgsfit_visibilities(
            dptr(u), dptr(v), dptr(w), dptr(x), N, Nbase, tilesz, barr, sky.arr, cptr(coh),
            sky.M, sky.Mt, freq0, fdelta, dptr(pp), uvmin, Nt, max_lbfgs, lbfgs_m, gpu_threads,
            solver_mode, mean_nu, C.byref(res0), C.byref(res1))
        return rv, res0.value, res1.value

    # ---- multi-channel minibatch LBFGS (Dirac.h:86-147,317-350) ----
    def persist_init(self, nminibatch, m, n, lbfgs_m, Nt=4):
        """a persistent_data_t owned by THIS library (the struct's layout is the library's business:
        a generous buffer takes either of the reference's two layouts)"""
        pt = C.create_string_buffer(1024)
        self.lib.lbfgs_persist_init(pt, nminibatch, m, n, lbfgs_m, Nt)
        return pt

    def persist_clear(self, pt):
        self.lib.lbfgs_persist_clear(pt)

    def bfgsfit_minibatch(self, u, v, w, x, N, Nbase, tilesz, barr, sky, coh, pp, freqs, pt,
                          fdelta=195.3e3, Nt=4, max_lbfgs=4, lbfgs_m=5, robust_nu=5.0, nmb=0,
                          totalmb=1, Y=None, Z=None, rho=None):
        """bfgsfit_minibatch_visibilities, or _consensus when Y / Z / rho are given.  x:
        [chan][row][8], coh: [chan][row][M][4] complex.  returns (res_0, res_1); pp in/out"""
        r0, r1 = C.c_double(0.0), C.c_double(0.0)
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        head = (dptr(u), dptr(v), dptr(w), dptr(x), N, Nbase, tilesz, barr, sky.arr, cptr(coh),
                sky.M, sky.Mt, dptr(freqs), len(freqs), C.c_double(fdelta), dptr(pp))
        tail = (Nt, max_lbfgs, lbfgs_m, 128, 2, C.c_double(robust_nu), C.byref(r0), C.byref(r1), pt,
                nmb, totalmb)
        if Y is None:
            self.lib.bfgsfit_minibatch_visibilities(*head, *tail)
        else:
            self.lib.bfgsfit_minibatch_consensus(*head, dptr(Y), dptr(Z), dptr(rho), *tail)
        return r0.value, r1.value

    @staticmethod
    def _interval_fn(L, name, argtypes, beam, nmb, tmb):
        """the interval call `name`, or its _withbeam variant with the beam arguments inserted after
        uvmax (the 17th argument) when beam is given; returns (function, beam arguments)"""
        if beam is None:
            fn = getattr(L, name)
            fn.restype, fn.argtypes = C.c_int, argtypes
            return fn, ()
        assert beam.tilesz == nmb * tmb, "time_utc is [minibatches][tmb]"
        dpp = C.POINTER(c_double_p)
        fn = getattr(L, name + "_withbeam")
        fn.restype = C.c_int
        fn.argtypes = argtypes[:17] + [C.c_int] + [C.c_double] * 5 + [c_double_p] * 3 + [
            c_int_p, dpp, dpp, dpp, C.POINTER(elementcoeff), C.c_int] + argtypes[17:]
        return fn, (*beam.head(), *beam.tail())

    def stochastic_interval(self, u, v, w, xo, N, Nbase, tmb, barr, sky: SkyModel, freqs, deltaf, pt,
                            pfreq, nsolbw, nepochs, uvmin=0.0, uvmax=1e9, max_lbfgs=4, lbfgs_m=5,
                            robust_nu=2.0, ccid=-99999, rho=1e-9, phase_only=0,
                            beam: "BeamSetup" = None):
        """dirac_b200_stochastic_interval: the minibatch driver's loop over one interval in one call.
        u, v, w [minibatches, Nbase*tmb]; xo [minibatches, Nchan, Nbase*tmb*8] data -> residual (in
        place); barr: minibatches * Nbase*tmb rows (input only); pt: nsolbw persistent_data_t
        (persist_init_array); pfreq [nsolbw, 8 N Mt] start -> solutions (in
        place); beam: station beams through dirac_b200_stochastic_interval_withbeam, its time_utc
        [minibatches][tmb].  returns (retval, res_00, res_01), each [nepochs, minibatches, nsolbw]"""
        for a in (u, v, w, xo, pfreq):
            assert a.dtype == np.float64 and a.flags.c_contiguous
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        nmb = u.shape[0]
        fn, bargs = self._interval_fn(self.lib, "dirac_b200_stochastic_interval", [c_double_p] * 4 + [
            C.c_int] * 4 + [
            C.POINTER(baseline_t), C.POINTER(clus_source_t), C.c_int, C.c_int, c_double_p, C.c_int,
            C.c_double, C.c_double, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double,
            C.c_void_p, c_double_p, C.c_int, C.c_double, C.c_int, c_double_p, c_double_p], beam, nmb,
            tmb)
        r0 = np.zeros((nepochs, nmb, nsolbw))
        r1 = np.zeros((nepochs, nmb, nsolbw))
        rv = fn(
            dptr(u), dptr(v), dptr(w), dptr(xo), N, Nbase, tmb, nmb, barr, sky.arr, sky.M, sky.Mt,
            dptr(freqs), len(freqs), deltaf, uvmin, uvmax, *bargs, nsolbw, nepochs, max_lbfgs,
            lbfgs_m, robust_nu, C.cast(pt, C.c_void_p), dptr(pfreq), ccid, rho, phase_only, dptr(r0),
            dptr(r1))
        return rv, r0, r1

    def stochastic_consensus_interval(self, u, v, w, xo, N, Nbase, tmb, barr, sky: SkyModel, freqs,
                                      deltaf, pt, pfreq, nsolbw, nepochs, nadmm, B, Bi, rhok, Z,
                                      use_global=0, uvmin=0.0, uvmax=1e9, max_lbfgs=4, lbfgs_m=5,
                                      robust_nu=2.0, ccid=-99999, rho=1e-9, phase_only=0,
                                      beam: "BeamSetup" = None):
        """dirac_b200_stochastic_consensus_interval: the consensus minibatch driver's loop over one
        interval in one call.  Arguments as stochastic_interval, plus B [nsolbw, Npoly],
        Bi [Mt, Npoly, Npoly], rhok [nsolbw, Mt] and Z [Mt, Npoly, 8N] (in place); beam: station
        beams through the _withbeam variant.  returns
        (retval, res_00, res_01 [nadmm, nepochs, minibatches, nsolbw], res_0, res_1, fband [nsolbw])"""
        dp, i, d = c_double_p, C.c_int, C.c_double
        fn, bargs = self._interval_fn(self.lib, "dirac_b200_stochastic_consensus_interval", [dp] * 4 + [
            i] * 4 + [
            C.POINTER(baseline_t), C.POINTER(clus_source_t), i, i, dp, i, d, d, d, i, i, i, i, d,
            C.c_void_p, dp, i, d, i, i, i, dp, dp, dp, dp, i, dp, dp, dp, dp, c_int_p], beam,
            u.shape[0], tmb)
        for a in (u, v, w, xo, pfreq, Z):
            assert a.dtype == np.float64 and a.flags.c_contiguous
        freqs = np.ascontiguousarray(freqs, dtype=np.float64)
        B = np.ascontiguousarray(B, dtype=np.float64)
        Bi = np.ascontiguousarray(Bi, dtype=np.float64)
        rhok = np.ascontiguousarray(rhok, dtype=np.float64)
        nmb = u.shape[0]
        r00 = np.zeros((nadmm, nepochs, nmb, nsolbw))
        r01 = np.zeros((nadmm, nepochs, nmb, nsolbw))
        r0, r1 = C.c_double(0.0), C.c_double(0.0)
        fband = np.zeros(max(nsolbw, 1), dtype=np.int32)
        rv = fn(
            dptr(u), dptr(v), dptr(w), dptr(xo), N, Nbase, tmb, nmb, barr, sky.arr, sky.M, sky.Mt,
            dptr(freqs), len(freqs), deltaf, uvmin, uvmax, *bargs, nsolbw, nepochs, max_lbfgs, lbfgs_m,
            robust_nu, C.cast(pt, C.c_void_p), dptr(pfreq), ccid, rho, phase_only, nadmm, B.shape[1],
            dptr(B), dptr(Bi), dptr(rhok), dptr(Z), use_global, dptr(r00), dptr(r01), C.byref(r0),
            C.byref(r1), fband.ctypes.data_as(c_int_p))
        return rv, r00, r01, r0.value, r1.value, fband[:nsolbw]

    def consensus_bands_update(self, N, res_00, res_01, pfreq, B, Bi, rhok, res_0, res_1, Y, Z):
        """dirac_b200_consensus_bands_update: the ADMM step after the bands of one minibatch.
        pfreq, Y [nsolbw, 8 N Mt]; B [nsolbw, Npoly]; Bi [Mt, Npoly, Npoly]; rhok [nsolbw, Mt];
        Z [Mt, Npoly, 8N].  Y and Z in place; returns (retval, res_0, res_1, fband)"""
        L = self.lib
        dp = c_double_p
        L.dirac_b200_consensus_bands_update.restype = C.c_int
        L.dirac_b200_consensus_bands_update.argtypes = [C.c_int] * 4 + [dp] * 6 + [dp, dp, dp, dp,
                                                                                 c_int_p]
        nsolbw, Npoly = B.shape
        Mt = Bi.shape[0]
        for a in (Y, Z):
            assert a.dtype == np.float64 and a.flags.c_contiguous
        r00 = np.ascontiguousarray(res_00, dtype=np.float64)
        r01 = np.ascontiguousarray(res_01, dtype=np.float64)
        args = [np.ascontiguousarray(a, dtype=np.float64) for a in (pfreq, B, Bi, rhok)]
        r0, r1 = C.c_double(res_0), C.c_double(res_1)
        fband = np.zeros(max(nsolbw, 1), dtype=np.int32)
        rv = L.dirac_b200_consensus_bands_update(N, Mt, nsolbw, Npoly, dptr(r00), dptr(r01),
                                                 *[dptr(a) for a in args], C.byref(r0), C.byref(r1),
                                                 dptr(Y), dptr(Z), fband.ctypes.data_as(c_int_p))
        return rv, r0.value, r1.value, fband[:nsolbw]

    def persist_init_array(self, nbands, nminibatch, m, n, lbfgs_m, Nt=4):
        """nbands persistent_data_t of include/dirac_b200.h back to back, as the driver's
        ptdata_array, each initialised by lbfgs_persist_init"""
        arr = (persistent_data_t * nbands)()
        for b in range(nbands):
            self.lib.lbfgs_persist_init(C.byref(arr[b]), nminibatch, m, n, lbfgs_m, Nt)
        return arr

    def sagefit_visibilities_admm(self, u, v, w, x, N, Nbase, tilesz, barr, sky, coh, pp, Y, BZ, rho,
                                  max_emiter=3, max_iter=2, nulow=2.0, nuhigh=30.0, Nt=4,
                                  solver_mode=5):
        """sagefit_visibilities_admm (Dirac.h:1521, admm_solve.c:221): x -> residual, pp in/out"""
        nu, r0, r1 = C.c_double(0), C.c_double(0), C.c_double(0)
        self.lib.sagefit_visibilities_admm.restype = C.c_int
        rv = self.lib.sagefit_visibilities_admm(
            dptr(u), dptr(v), dptr(w), dptr(x), N, Nbase, tilesz, barr, sky.arr, cptr(coh), sky.M,
            sky.Mt, C.c_double(150e6), C.c_double(195.3e3), dptr(pp), dptr(Y), dptr(BZ),
            C.c_double(0.0), Nt, max_emiter, max_iter, 0, 7, 128, 0, solver_mode, C.c_double(nulow),
            C.c_double(nuhigh), 0, dptr(rho), C.byref(nu), C.byref(r0), C.byref(r1))
        return rv, nu.value, r0.value, r1.value

