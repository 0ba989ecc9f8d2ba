"""Stochastic calibration of one interval with station beams (sagecal -N 2 -M 4 -w 2 -B 5,
minibatch_mode.cpp:364-509 with its beam branches) at the shape of profiles/stochastic.py: 62 stations,
64 clusters, 120 timeslots in 4 minibatches of 30, 8 channels in 2 bands, 2 epochs, robust nu 2, from a
perturbed start, corrected by one cluster.  The beam is DOBEAM_FULL_WB with a tile beam-former of
HBA-like size (16 dipoles per tile, 24-48 tiles per station), on seeded synthetic station layouts and
seeded synthetic element coefficient tables of the reference's sizes (model order 7, 28 modes, one set
per channel).  Times (a) dirac_b200_stochastic_interval_withbeam and (b) the driver's loop restated
with this library's reference-named calls (precalculate_coherencies_multifreq_withbeam per minibatch in
the first epoch, bfgsfit_minibatch_visibilities per epoch, minibatch and band,
calculate_residuals_multifreq_withbeam per minibatch and band, flags preset at every load), as wall
time of the calls (profiling off, best and all of --reps after a warm-up of each), alternating (a) and
(b); then, in one more repeat of each with profiling on, the CUDA-event time and launches of the beam
tables (k_beam_tables, kind 15), the interval's coherency prediction (kind 16), the band cost /
residual pass (k_stream_band, kind 13) and the band gradient (k_grad_tma_band, kind 14), the sky
uploads and the bytes of coherencies that crossed PCIe; and the largest difference of the two answers.
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; with
--out, writes it there too.

    python profiles/stochastic_beam.py [--reps 3] [--out FILE]"""
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
from sagecal_b200 import synth, lib as blib  # noqa: E402
from sagecal_b200.dirac_api import BeamSetup, SkyModel, elementcoeff, make_barr  # noqa: E402
from minibatch_stage import card, kernel_ms  # noqa: E402

KIND_BAND, KIND_BAND_GRAD, KIND_BEAM, KIND_COH = 13, 14, 15, 16
DOBEAM_FULL_WB, STAT_TILE = 5, 2
EC_M, EC_BETA = 7, 0.5
NMB, NCHAN, NBANDS, NEPOCHS = 4, 8, 2, 2
FIT = dict(max_lbfgs=10, lbfgs_m=7, robust_nu=2.0)
CORR = dict(ccid=3, rho=1e-9)


def synthetic_beam(pr, nmb, tmb, freqs, seed=11):
    """directions for every source near the phase centre, station positions, HBA-like tiles and one
    coefficient set per channel, all seeded; one BeamSetup for the interval ([nmb][tmb] JD) and one per
    minibatch.  The returned list keeps the buffers the tables point to alive."""
    rng = np.random.default_rng(seed)
    ra0, dec0 = 1.2, np.deg2rad(58.0)
    for cl in pr.clusters:
        K = len(cl["ll"])
        cl["ra"] = ra0 + np.deg2rad(rng.uniform(-5, 5, K))
        cl["dec"] = dec0 + np.deg2rad(rng.uniform(-5, 5, K))
    lon = np.deg2rad(6.87 + rng.uniform(-0.5, 0.5, pr.N))
    lat = np.deg2rad(52.9 + rng.uniform(-0.3, 0.3, pr.N))
    g = (np.arange(4) - 1.5) * 1.25
    dip = np.array([[x, y, 0.0] for x in g for y in g])
    elems = []
    for n in range(pr.N):
        nt = int(rng.integers(24, 49))
        elems.append(np.vstack([dip, np.c_[rng.uniform(-30, 30, (nt, 2)), rng.normal(0, 0.05, nt)]]))
    nmodes = EC_M * (EC_M + 1) // 2
    phi = rng.normal(0, 1, 2 * nmodes * len(freqs))
    theta = rng.normal(0, 1, 2 * nmodes * len(freqs))
    pre = rng.uniform(0.5, 1.5, nmodes)
    keep = [phi, theta, pre]
    ec = elementcoeff(EC_M, nmodes, len(freqs), EC_BETA, phi.ctypes.data, theta.ctypes.data,
                      pre.ctypes.data)
    t = 2456789.3 + np.arange(nmb * tmb) * 10.0 / 86400.0
    mk = lambda tt: BeamSetup(STAT_TILE, ra0 + 0.01, dec0 - 0.01, ra0, dec0, float(np.mean(freqs)), lon,
                              lat, tt, elems, ec, DOBEAM_FULL_WB)
    return mk(t), [mk(t[mb * tmb:(mb + 1) * tmb]) for mb in range(nmb)], keep + [ec]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--config", default="C3")
    ap.add_argument("--max-lbfgs", type=int, default=FIT["max_lbfgs"],
                    help="0: no LBFGS iterations, so that the two answers must agree to the last bits")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("stochastic.py measures on a GPU; none is visible")
    FIT["max_lbfgs"] = args.max_lbfgs
    api = blib.load()
    pr = synth.make_config(args.config)
    tmb = pr.tilesz // NMB
    R = pr.Nbase * tmb
    deltaf = pr.fdelta
    freqs = pr.freq0 + (np.arange(NCHAN) - 0.5 * (NCHAN - 1)) * deltaf / NCHAN
    per = (NCHAN + NBANDS - 1) // NBANDS
    bands = [(b * per, min(per, NCHAN - b * per)) for b in range(NBANDS)]
    beam, beam_mb, _keep = synthetic_beam(pr, NMB, tmb, freqs)
    sky = SkyModel(pr.clusters, pr.N)
    rng = np.random.default_rng(5)
    p0 = pr.pp0 + 0.02 * rng.normal(0, 1, pr.pp0.shape)
    sl = lambda a: np.ascontiguousarray(a[:NMB * R].reshape(NMB, R))
    u, v, w = sl(pr.u), sl(pr.v), sl(pr.w)
    sta1, sta2, flag = (a[:NMB * R].reshape(NMB, R) for a in (pr.sta1, pr.sta2, pr.flag))
    # data simulated through the same beams (predict_visibilities_multifreq_withsol_withbeam) with
    # Jones near the start, plus 1 % noise: a beam model fitted to beam-less data is a poorly posed
    # fit on which the last-bit differences of two runs grow
    ptrue = pr.pp0 + 0.05 * rng.normal(0, 1, pr.pp0.shape)
    xo0 = np.zeros((NMB, NCHAN, 8 * R))
    for mb in range(NMB):
        xs = np.zeros(NCHAN * 8 * R)
        api.predict_visibilities_multifreq_withsol_withbeam(
            u[mb], v[mb], w[mb], ptrue, xs, pr.N, pr.Nbase, tmb, make_barr(sta1[mb], sta2[mb], flag[mb]),
            sky, freqs, deltaf, beam_mb[mb])
        xs = xs.reshape(NCHAN, R, 8)
        xs += rng.normal(0, 0.01 * np.median(np.abs(xs)), xs.shape)
        xs[:, flag[mb] != 0] = 0.0   # preset_flags_and_data
        xo0[mb] = xs.reshape(NCHAN, 8 * R)
    m = len(p0)
    rep = {"shape": dict(N=pr.N, M=pr.M, Mt=pr.Mt, tilesz=pr.tilesz, minibatches=NMB, tmb=tmb,
                         Nchan=NCHAN, bands=NBANDS, epochs=NEPOCHS,
                         coherency_bytes=NMB * NCHAN * pr.M * R * 64,
                         sources=sum(len(cl["ll"]) for cl in pr.clusters), doBeam=DOBEAM_FULL_WB,
                         tiles_per_station=[int(n) for n in beam.Nelem], **FIT)}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()

    def interval():
        xo = xo0.copy()
        pfreq = np.tile(p0, (NBANDS, 1))
        pts = api.persist_init_array(NBANDS, NMB, m, 8 * R, FIT["lbfgs_m"])
        barr = make_barr(sta1.reshape(-1), sta2.reshape(-1), flag.reshape(-1))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rv, r0, r1 = api.stochastic_interval(u, v, w, xo, pr.N, pr.Nbase, tmb, barr, sky, freqs, deltaf,
                                            pts, pfreq, NBANDS, NEPOCHS, beam=beam, **FIT, **CORR)
        t = dict(total=time.perf_counter() - t0)
        assert rv == 0
        for b in range(NBANDS):
            api.lib.lbfgs_persist_clear(C.byref(pts[b]))
        return t, xo, pfreq, r1, r0

    def reference_named():
        xo = xo0.copy()
        pfreq = np.tile(p0, (NBANDS, 1))
        pts = [api.persist_init(NMB, m, 8 * R, FIT["lbfgs_m"]) for _ in range(NBANDS)]
        r1 = np.zeros((NEPOCHS, NMB, NBANDS))
        r0 = np.zeros((NEPOCHS, NMB, NBANDS))
        t = dict(precalculate=0.0, bfgsfit=0.0, residual=0.0)
        coh = [None] * NMB
        torch.cuda.synchronize()
        for ep in range(NEPOCHS):
            for mb in range(NMB):
                barr = make_barr(sta1[mb], sta2[mb], flag[mb])
                t0 = time.perf_counter()
                if ep == 0:
                    coh[mb] = api.precalculate_coherencies_multifreq(u[mb], v[mb], w[mb], pr.N, R, barr,
                                                                     sky, freqs, deltaf, beam_mb[mb])
                t1 = time.perf_counter()
                for b, (c0, nc) in enumerate(bands):
                    cb = coh[mb][c0 * R * pr.M * 4:(c0 + nc) * R * pr.M * 4]
                    xb = xo[mb, c0:c0 + nc].reshape(-1).copy()
                    r0[ep, mb, b], r1[ep, mb, b] = api.bfgsfit_minibatch(
                        u[mb], v[mb], w[mb], xb, pr.N, pr.Nbase, tmb, barr, sky, cb, pfreq[b],
                        freqs[c0:c0 + nc], pts[b], fdelta=deltaf / NCHAN * nc, nmb=mb, totalmb=NMB,
                        **FIT)
                t2 = time.perf_counter()
                t["precalculate"] += t1 - t0
                t["bfgsfit"] += t2 - t1
        t0 = time.perf_counter()
        for mb in range(NMB):
            barr = make_barr(sta1[mb], sta2[mb], flag[mb])
            for b, (c0, nc) in enumerate(bands):
                xr = np.ascontiguousarray(xo[mb, c0:c0 + nc])
                api.calculate_residuals_multifreq_withbeam(u[mb], v[mb], w[mb], pfreq[b],
                                                           xr.reshape(-1), pr.N, pr.Nbase, tmb, barr,
                                                           sky, freqs[c0:c0 + nc],
                                                           deltaf / NCHAN * nc, beam_mb[mb], **CORR)
                xo[mb, c0:c0 + nc] = xr
        t["residual"] = time.perf_counter() - t0
        t["total"] = sum(t.values())
        for pt in pts:
            api.persist_clear(pt)
        return t, xo, pfreq, r1, r0

    variants = (("interval", interval), ("reference_named", reference_named))
    out = {}
    for name, fn in variants:  # warm-up of every shape, and the two answers
        out[name] = fn()
    xa, xb = out["interval"][1], out["reference_named"][1]
    rep["interval_vs_reference_named"] = dict(
        residual_maxerr_over_max=float(np.max(np.abs(xa - xb)) / np.max(np.abs(xb))),
        jones_maxerr_over_max=float(np.max(np.abs(out["interval"][2] - out["reference_named"][2]))
                                    / np.max(np.abs(out["reference_named"][2]))),
        res_00_maxrelerr=float(np.max(np.abs(out["interval"][4] - out["reference_named"][4])
                                      / np.abs(out["reference_named"][4]))),
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
        for label, kind in (("beam_tables", KIND_BEAM), ("interval_coherencies", KIND_COH),
                            ("band_cost_or_residual", KIND_BAND), ("band_gradient", KIND_BAND_GRAD)):
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
