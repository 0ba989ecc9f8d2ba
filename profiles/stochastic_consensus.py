"""Stochastic calibration with spectral consensus over the bands for one interval (sagecal -N 2 -M 4 -w 4
-A 3, minibatch_consensus_mode.cpp:450-672) at a C3-like shape: 62 stations, 64 clusters, 120 timeslots
in 4 minibatches of 30, 8 channels in 4 bands, 3 ADMM iterations of 2 epochs, Npoly 2, PolyType 2
(Bernstein), ADMM rho 5, robust nu 2, from a perturbed start, corrected by one cluster.  Times (a)
dirac_b200_stochastic_consensus_interval and (b) the driver's loop restated with the reference-named
calls (precalculate_coherencies_multifreq per minibatch in the first pass, bfgsfit_minibatch_consensus
per ADMM iteration, epoch, minibatch and band, dirac_b200_consensus_bands_update per minibatch,
calculate_residuals_multifreq per minibatch and band, flags preset at every load), as wall time of the
calls (profiling off, best and all of --reps after a warm-up of each), alternating (a) and (b); then, in
one more repeat of each with profiling on, the CUDA-event time of the band cost / residual pass
(k_stream_band, kind 13) and the band gradient (k_grad_tma_band, kind 14), the launches of each per
cost and gradient evaluation, the sky uploads and the bytes of coherencies that crossed PCIe; and the
largest difference of the two answers.  The card's name, power limit and maximum SM clock are read in
the same run.  Prints one JSON line; with --out, writes it there too.

    python profiles/stochastic_consensus.py [--reps 3] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sagecal_b200 import consensus as cons, synth, lib as blib  # noqa: E402
from sagecal_b200.dirac_api import SkyModel, make_barr  # noqa: E402
from minibatch_stage import card, kernel_ms  # noqa: E402

KIND_BAND, KIND_BAND_GRAD = 13, 14
NMB, NCHAN, NBANDS, NEPOCHS, NADMM, NPOLY, POLYTYPE, ADMM_RHO = 4, 8, 4, 2, 3, 2, 2, 5.0
FIT = dict(max_lbfgs=10, lbfgs_m=7, robust_nu=2.0)
CORR = dict(ccid=3, rho=1e-9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--config", default="C3")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("stochastic_consensus.py measures on a GPU; none is visible")
    api = blib.load()
    pr = synth.make_config(args.config)
    sky = SkyModel(pr.clusters, pr.N)
    tmb = pr.tilesz // NMB
    R = pr.Nbase * tmb
    deltaf = pr.fdelta
    freqs = pr.freq0 + (np.arange(NCHAN) - 0.5 * (NCHAN - 1)) * deltaf / NCHAN
    per = (NCHAN + NBANDS - 1) // NBANDS
    bands = [(b * per, min(per, NCHAN - b * per)) for b in range(NBANDS)]
    rng = np.random.default_rng(5)
    p0 = pr.pp0 + 0.02 * rng.normal(0, 1, pr.pp0.shape)
    sl = lambda a: np.ascontiguousarray(a[:NMB * R].reshape(NMB, R))
    u, v, w = sl(pr.u), sl(pr.v), sl(pr.w)
    sta1, sta2, flag = (a[:NMB * R].reshape(NMB, R) for a in (pr.sta1, pr.sta2, pr.flag))
    x0 = pr.x[:NMB * R * 8].reshape(NMB, 1, 8 * R)
    xo0 = np.ascontiguousarray(np.concatenate([x0 * (1.0 + 0.01 * c) for c in range(NCHAN)], axis=1))
    m = len(p0)
    B = cons.basis(api, np.array([freqs[c0:c0 + nc].mean() for c0, nc in bands]), pr.freq0, NPOLY,
                   POLYTYPE)
    rhok = np.full((NBANDS, pr.Mt), ADMM_RHO)
    Bi = cons.prod_inverse(api, B, rhok)
    rep = {"shape": dict(N=pr.N, M=pr.M, Mt=pr.Mt, tilesz=pr.tilesz, minibatches=NMB, tmb=tmb,
                         Nchan=NCHAN, bands=NBANDS, epochs=NEPOCHS, nadmm=NADMM, Npoly=NPOLY,
                         PolyType=POLYTYPE, admm_rho=ADMM_RHO,
                         coherency_bytes=NMB * NCHAN * pr.M * R * 64, **FIT)}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()

    def interval():
        xo = xo0.copy()
        pfreq = np.tile(p0, (NBANDS, 1))
        pts = api.persist_init_array(NBANDS, NMB, m, 8 * R, FIT["lbfgs_m"])
        Z = np.zeros((pr.Mt, NPOLY, 8 * pr.N))
        barr = make_barr(sta1.reshape(-1), sta2.reshape(-1), flag.reshape(-1))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rv, _, r1, _, _, _ = api.stochastic_consensus_interval(
            u, v, w, xo, pr.N, pr.Nbase, tmb, barr, sky, freqs, deltaf, pts, pfreq, NBANDS, NEPOCHS,
            NADMM, B, Bi, rhok, Z, **FIT, **CORR)
        t = dict(total=time.perf_counter() - t0)
        assert rv == 0
        for b in range(NBANDS):
            api.lib.lbfgs_persist_clear(C.byref(pts[b]))
        return t, xo, pfreq, r1[-1]

    def reference_named():
        xo = xo0.copy()
        pfreq = np.tile(p0, (NBANDS, 1))
        pts = [api.persist_init(NMB, m, 8 * R, FIT["lbfgs_m"]) for _ in range(NBANDS)]
        r1 = np.zeros((NEPOCHS, NMB, NBANDS))
        r0 = np.zeros((NEPOCHS, NMB, NBANDS))
        Y = np.zeros((NBANDS, m))
        Z = np.zeros((pr.Mt, NPOLY, 8 * pr.N))
        res_0 = res_1 = 0.0
        t = dict(precalculate=0.0, bfgsfit=0.0, admm=0.0, residual=0.0)
        coh = [None] * NMB
        torch.cuda.synchronize()
        for ad in range(NADMM):
            for ep in range(NEPOCHS):
                for mb in range(NMB):
                    barr = make_barr(sta1[mb], sta2[mb], flag[mb])
                    t0 = time.perf_counter()
                    if ep == 0 and ad == 0:
                        coh[mb] = api.precalculate_coherencies_multifreq(u[mb], v[mb], w[mb], pr.N, R,
                                                                         barr, sky, freqs, deltaf)
                    t1 = time.perf_counter()
                    for b, (c0, nc) in enumerate(bands):
                        z = np.einsum("p,kpi->ki", B[b], Z).reshape(-1)
                        cb = coh[mb][c0 * R * pr.M * 4:(c0 + nc) * R * pr.M * 4]
                        xb = xo[mb, c0:c0 + nc].reshape(-1).copy()
                        r0[ep, mb, b], r1[ep, mb, b] = api.bfgsfit_minibatch(
                            u[mb], v[mb], w[mb], xb, pr.N, pr.Nbase, tmb, barr, sky, cb, pfreq[b],
                            freqs[c0:c0 + nc], pts[b], fdelta=deltaf / NCHAN * nc, nmb=mb,
                            totalmb=NMB, Y=Y[b], Z=z, rho=np.ascontiguousarray(rhok[b]), **FIT)
                    t2 = time.perf_counter()
                    rv, res_0, res_1, _ = api.consensus_bands_update(pr.N, r0[ep, mb], r1[ep, mb], pfreq,
                                                                     B, Bi, rhok, res_0, res_1, Y, Z)
                    assert rv == 0
                    t["precalculate"] += t1 - t0
                    t["bfgsfit"] += t2 - t1
                    t["admm"] += time.perf_counter() - t2
        t0 = time.perf_counter()
        for mb in range(NMB):
            barr = make_barr(sta1[mb], sta2[mb], flag[mb])
            for b, (c0, nc) in enumerate(bands):
                xr = np.ascontiguousarray(xo[mb, c0:c0 + nc])
                api.calculate_residuals_multifreq(u[mb], v[mb], w[mb], pfreq[b], xr.reshape(-1), pr.N,
                                                  pr.Nbase, tmb, barr, sky, freqs[c0:c0 + nc],
                                                  deltaf / NCHAN * nc, **CORR)
                xo[mb, c0:c0 + nc] = xr
        t["residual"] = time.perf_counter() - t0
        t["total"] = sum(t.values())
        for pt in pts:
            api.persist_clear(pt)
        return t, xo, pfreq, r1

    variants = (("interval", interval), ("reference_named", reference_named))
    out = {}
    for name, fn in variants:  # warm-up of every shape, and the two answers
        out[name] = fn()
    xa, xb = out["interval"][1], out["reference_named"][1]
    rep["interval_vs_reference_named"] = dict(
        residual_maxerr_over_max=float(np.max(np.abs(xa - xb)) / np.max(np.abs(xb))),
        jones_maxerr_over_max=float(np.max(np.abs(out["interval"][2] - out["reference_named"][2]))
                                    / np.max(np.abs(out["reference_named"][2]))),
        res_01_last_epoch=[out["interval"][3][-1].tolist(), out["reference_named"][3][-1].tolist()])
    walls = {name: [] for name, _ in variants}
    for _ in range(args.reps):
        for name, fn in variants:
            walls[name].append(fn()[0])
    for name, _ in variants:
        tot = [1e3 * wl["total"] for wl in walls[name]]
        best = walls[name][int(np.argmin(tot))]
        rep[name] = dict(call_ms_min=min(tot), call_ms_all=tot,
                         split_ms_of_min={k: 1e3 * val for k, val in best.items() if k != "total"})
    for name, fn in variants:  # kernel times, launches and traffic, in a run of their own
        api.transfer_stats(reset=True)
        k13, k14 = api.kernel_count(KIND_BAND), api.kernel_count(KIND_BAND_GRAD)
        api.profile_enable(True)
        fn()
        for label, kind in (("band_cost_or_residual", KIND_BAND), ("band_gradient", KIND_BAND_GRAD)):
            nk, ms, _ = kernel_ms(api, kind)
            rep[name][label] = dict(launches=nk, ms_total=ms)
        api.profile_enable(False)
        ngrad = api.kernel_count(KIND_BAND_GRAD) - k14
        ncost = api.kernel_count(KIND_BAND) - k13 - ngrad
        rep[name]["evaluations"] = dict(cost=ncost, gradient=ngrad)
        up, by = api.transfer_stats(reset=True)
        rep[name]["sky_uploads"], rep[name]["coherency_bytes_over_pcie"] = up, by
    line = json.dumps(rep)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
