"""Full-batch calibration of one tile (dirac_b200_fullbatch_tile(_withbeam)) against the driver's chain of
reference-named calls (precalculate_coherencies(_withbeam) -> sagefit_visibilities ->
calculate_residuals_multifreq(_withbeam)) at the C2 shape: 62 stations, 64 clusters, 120 timeslots, 8
channels, solver_mode 1 and 5, without beam and with the wide-band full beam (DOBEAM_FULL_WB; element
coefficients from the compiled reference's set_elementcoeffs_wb, oracle/_ref).  Per case, best of --reps
host wall times of each, the sky uploads and coherency bytes over PCIe, the CUDA-event times of the
tile's coherencies (profile kind 24), fit (25), beam tables (15) and residual (11), and the largest
output differences.  The card's name, power limit and maximum SM clock are read in the same run.  Prints
one JSON line; with --out, writes it there too.

    python profiles/fullbatch.py [--reps 3] [--out FILE]"""
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
from sagecal_b200.dirac_api import BeamSetup, SkyModel, elementcoeff, dptr, make_barr  # noqa: E402
from minibatch_stage import card  # noqa: E402

NCHAN = 8
KINDS = {"coherencies": 24, "fit": 25, "beam_tables": 15, "residual": 11}


def full_wb_beam(pr, freqs):
    """stations, elements, timeslots and source directions of test_gpu_beam.py's construction"""
    import refdirac
    rng = np.random.default_rng(31)
    ra0, dec0 = 1.2, np.deg2rad(58.0)
    for cl in pr.clusters:
        K = len(cl["ll"])
        cl["ra"] = ra0 + np.deg2rad(rng.uniform(-4, 4, K))
        cl["dec"] = dec0 + np.deg2rad(rng.uniform(-4, 4, K))
    elems = [np.c_[rng.uniform(-40, 40, (40 + n % 8, 2)), rng.normal(0, 0.1, 40 + n % 8)]
             for n in range(pr.N)]
    ec = elementcoeff()
    ref = refdirac.RefDirac()
    f = np.ascontiguousarray(freqs, dtype=np.float64)
    ref.lib.set_elementcoeffs_wb(0, dptr(f), len(f), C.byref(ec))
    t = 2456789.3 + np.arange(pr.tilesz) * 10.0 / 86400.0
    return BeamSetup(1, ra0 + 0.01, dec0 - 0.01, ra0, dec0, float(np.mean(freqs)),
                     np.deg2rad(6.87 + rng.uniform(-0.5, 0.5, pr.N)),
                     np.deg2rad(52.9 + rng.uniform(-0.3, 0.3, pr.N)), t, elems, ec, 5), ref


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("fullbatch.py measures on a GPU; none is visible")
    api = blib.load()
    pr = synth.make_config("C2")
    freqs = pr.freq0 + (np.arange(NCHAN) - NCHAN / 2 + 0.5) * pr.fdelta
    deltaf = pr.fdelta * NCHAN
    rng = np.random.default_rng(7)
    xo0 = np.ascontiguousarray(np.stack([pr.x + rng.normal(0, 1e-3, pr.x.shape) for _ in freqs]))
    x0 = np.ascontiguousarray(xo0.mean(axis=0))
    rep = {"shape": dict(N=pr.N, Nbase=pr.Nbase, M=pr.M, Mt=pr.Mt, tilesz=pr.tilesz, Nchan=NCHAN)}
    rep["card"], rep["power_limit_and_max_sm_clock"] = card()
    beam, keep = full_wb_beam(pr, freqs)
    sky = SkyModel(pr.clusters, pr.N)
    fit = dict(max_emiter=3, max_iter=2, max_lbfgs=10, lbfgs_m=7)
    cases = []
    for mode in (1, 5):
        for bm in (None, beam):
            kw = dict(fit, solver_mode=mode)
            barr = lambda: make_barr(pr.sta1, pr.sta2, pr.flag)

            def chain():
                x, xo, p, b = x0.copy(), xo0.copy(), pr.pp0.copy(), barr()
                if bm is None:
                    coh = api.precalculate_coherencies(pr.u, pr.v, pr.w, pr.N, pr.Nbase1, b, sky,
                                                       pr.freq0, deltaf)
                else:
                    coh = api.precalculate_coherencies_withbeam(pr.u, pr.v, pr.w, pr.N, pr.Nbase1, b,
                                                                sky, pr.freq0, deltaf, bm)
                api.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, b, sky, coh, p,
                                         freq0=pr.freq0, fdelta=deltaf, **kw)
                if bm is None:
                    api.calculate_residuals_multifreq(pr.u, pr.v, pr.w, p, xo, pr.N, pr.Nbase, pr.tilesz,
                                                      b, sky, freqs, deltaf, ccid=1)
                else:
                    api.calculate_residuals_multifreq_withbeam(pr.u, pr.v, pr.w, p, xo, pr.N, pr.Nbase,
                                                               pr.tilesz, b, sky, freqs, deltaf, bm,
                                                               ccid=1)
                return x, xo, p

            def tile():
                x, xo, p = x0.copy(), xo0.copy(), pr.pp0.copy()
                rv = api.fullbatch_tile(pr.u, pr.v, pr.w, x, xo, pr.N, pr.Nbase, pr.tilesz, barr(), sky,
                                        pr.freq0, deltaf, freqs, p, ccid=1, beam=bm, **kw)[0]
                assert rv == 0
                return x, xo, p

            res = {"solver_mode": mode, "beam": "none" if bm is None else "DOBEAM_FULL_WB"}
            for name, fn in (("chain", chain), ("tile", tile)):
                fn()   # warm-up: modules, cuSOLVER, the allocator's cache
                walls, io = [], None
                for r in range(args.reps):
                    api.transfer_stats(reset=True)
                    if name == "tile":
                        api.lib.dirac_b200_profile_enable(1)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    out = fn()
                    walls.append(time.perf_counter() - t0)
                    io = api.transfer_stats(reset=True)
                    if name == "tile" and r == args.reps - 1:
                        ms = C.c_double(0.0)
                        for k, kind in KINDS.items():
                            n = api.lib.dirac_b200_profile_read(kind, C.byref(ms), None)
                            res["tile_%s_ms" % k] = round(ms.value, 2) if n else None
                    api.lib.dirac_b200_profile_enable(0)
                res[name + "_wall_ms_best"] = round(1e3 * min(walls), 1)
                res[name + "_sky_uploads"], res[name + "_coh_pcie_bytes"] = io
                res[name + "_out"] = out
            (cx, cxo, cp), (tx, txo, tp) = res.pop("chain_out"), res.pop("tile_out")
            rel = lambda a, b: float(np.max(np.abs(a - b)) / np.max(np.abs(b)))
            res["maxdiff_rel"] = dict(x=rel(tx, cx), xo=rel(txo, cxo), p=rel(tp, cp))
            cases.append(res)
    del keep
    rep["cases"] = cases
    line = json.dumps(rep)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
