"""Per-channel refinement (driver option -b 1) at the C3 shape: 62 stations, 64 clusters, 120 timeslots,
8 channels, robust LBFGS (solver_mode 2) from a perturbed start, corrected by one cluster.  Times
(a) dirac_b200_bfgsfit_channels, the whole channel loop on one resident problem, and (b) the same loop
through precalculate_coherencies, bfgsfit_visibilities and calculate_residuals per channel, as wall time
of the calls (profiling off, best and all of --reps after a warm-up of each), alternating (a) and (b);
then, in one more repeat of each with profiling on, the CUDA-event time of the all-cluster predict pass
(kind 0) and of the residual from the sky (k_sky_predict<2>, kind 11); the sky uploads and the bytes of
coherencies that crossed PCIe per loop; the largest difference of the two loops' answers; and, if
oracle/_ref is built, (c) the reference's CPU calculate_residuals of one channel with all host threads.
The card's name, power limit and maximum SM clock are read in the same run.  Prints one JSON line; with
--out, writes it there too.

    python profiles/perchannel.py [--reps 3] [--channels 8] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sagecal_b200 import synth, lib as blib  # noqa: E402
from sagecal_b200.dirac_api import SkyModel, make_barr  # noqa: E402
from minibatch_stage import card, kernel_ms  # noqa: E402

KIND_PREDICT, KIND_SKY_RESIDUAL = 0, 11
FIT = dict(max_lbfgs=10, lbfgs_m=7, solver_mode=2, mean_nu=2.0)
CORR = dict(ccid=3, rho=1e-9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--channels", type=int, default=8)
    ap.add_argument("--config", default="C3")
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("perchannel.py measures on a GPU; none is visible")
    api = blib.load()
    api.lib.dirac_b200_profile_enable.argtypes = [C.c_int]
    pr = synth.make_config(args.config)
    sky = SkyModel(pr.clusters, pr.N)
    nch = args.channels
    deltafch = pr.fdelta / nch
    freqs = pr.freq0 + (np.arange(nch) - 0.5 * (nch - 1)) * deltafch
    rng = np.random.default_rng(5)
    p0 = pr.pp0 + 0.02 * rng.normal(0, 1, pr.pp0.shape)
    xo0 = np.stack([pr.x * (1.0 + 0.01 * c) for c in range(nch)])
    rep = {"shape": dict(N=pr.N, M=pr.M, Mt=pr.Mt, tilesz=pr.tilesz, rows=pr.Nbase1, Nchan=nch,
                         sources=int(sum(len(c["ll"]) for c in pr.clusters)), **FIT)}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()

    def resident():
        xo, p = xo0.copy(), p0.copy()
        barr = make_barr(pr.sta1, pr.sta2, pr.flag)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rv, r0, r1, _ = api.bfgsfit_channels(pr.u, pr.v, pr.w, xo.reshape(-1), pr.N, pr.Nbase, pr.tilesz,
                                             barr, sky, freqs, deltafch, p, keep_pfreq=False, **FIT,
                                             **CORR)
        assert rv == 0
        return dict(total=time.perf_counter() - t0), xo, p, r1

    def three_calls():
        xo, p = xo0.copy(), p0.copy()
        barr = make_barr(pr.sta1, pr.sta2, pr.flag)
        t = dict(precalculate=0.0, bfgsfit=0.0, residual=0.0)
        r1 = np.zeros(nch)
        torch.cuda.synchronize()
        for ci in range(nch):
            pf, xf = p0.copy(), xo[ci].copy()
            t0 = time.perf_counter()
            coh = api.precalculate_coherencies(pr.u, pr.v, pr.w, pr.N, pr.Nbase1, barr, sky, freqs[ci],
                                               deltafch)
            t1 = time.perf_counter()
            _, _, r1[ci] = api.bfgsfit_visibilities(pr.u, pr.v, pr.w, xf, pr.N, pr.Nbase, pr.tilesz, barr,
                                                    sky, coh, pf, freq0=freqs[ci], fdelta=deltafch, **FIT)
            t2 = time.perf_counter()
            api.calculate_residuals(pr.u, pr.v, pr.w, pf, xo[ci], pr.N, pr.Nbase, pr.tilesz, barr, sky,
                                    freqs[ci], deltafch, **CORR)
            t3 = time.perf_counter()
            t["precalculate"] += t1 - t0
            t["bfgsfit"] += t2 - t1
            t["residual"] += t3 - t2
            p = pf
        t["total"] = sum(t.values())
        return t, xo, p, r1

    variants = (("resident", resident), ("three_calls", three_calls))
    out = {}
    for name, fn in variants:  # warm-up of every shape, and the two answers
        out[name] = fn()
    xa, xb = out["resident"][1], out["three_calls"][1]
    rep["resident_vs_three_calls"] = dict(
        residual_maxerr_over_max=float(np.max(np.abs(xa - xb)) / np.max(np.abs(xb))),
        jones_maxerr_over_max=float(np.max(np.abs(out["resident"][2] - out["three_calls"][2]))
                                    / np.max(np.abs(out["three_calls"][2]))),
        res_01=[out["resident"][3].tolist(), out["three_calls"][3].tolist()])
    walls = {name: [] for name, _ in variants}
    for _ in range(args.reps):
        for name, fn in variants:
            walls[name].append(fn()[0])
    for name, _ in variants:
        tot = [1e3 * w["total"] for w in walls[name]]
        best = walls[name][int(np.argmin(tot))]
        rep[name] = dict(call_ms_min=min(tot), call_ms_all=tot,
                         split_ms_of_min={k: 1e3 * v for k, v in best.items() if k != "total"})
    for name, fn in variants:  # kernel times and traffic, in a run of their own
        api.transfer_stats(reset=True)
        api.lib.dirac_b200_profile_enable(1)
        fn()
        for label, kind in (("predict_pass", KIND_PREDICT), ("sky_residual", KIND_SKY_RESIDUAL)):
            nk, ms, _ = kernel_ms(api, kind)
            rep[name][label] = dict(launches=nk, ms_total=ms)
        api.lib.dirac_b200_profile_enable(0)
        up, by = api.transfer_stats(reset=True)
        rep[name]["sky_uploads"], rep[name]["coherency_bytes_over_pcie"] = up, by

    import refdirac
    if refdirac.available():
        nt = os.cpu_count() or 1
        x = xo0[0].copy()
        barr = make_barr(pr.sta1, pr.sta2, pr.flag)
        t0 = time.perf_counter()
        refdirac.load().calculate_residuals(pr.u, pr.v, pr.w, p0, x, pr.N, pr.Nbase, pr.tilesz, barr, sky,
                                            freqs[0], deltafch, Nt=nt, **CORR)
        rep["reference_cpu_residual_one_channel_ms"] = 1e3 * (time.perf_counter() - t0)
        rep["reference_threads"] = nt
        y = xo0[0].copy()
        api.calculate_residuals(pr.u, pr.v, pr.w, p0, y, pr.N, pr.Nbase, pr.tilesz,
                                make_barr(pr.sta1, pr.sta2, pr.flag), sky, freqs[0], deltafch, **CORR)
        rep["residual_relerr_vs_reference"] = float(np.max(np.abs(y - x)) / np.max(np.abs(x)))
    else:
        rep["reference_cpu_residual_one_channel_ms"] = "not measured (oracle/_ref not built)"
    line = json.dumps(rep)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
