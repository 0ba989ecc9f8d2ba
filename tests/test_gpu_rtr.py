"""GPU parity of solver_mode 4 (RSD + RTR), 5 (robust RTR, the reference driver's default) and 6
(Nesterov) through the drop-in entry point, against the compiled reference CPU path.  The robust
modes are compared with the reference build whose worker threads run synchronously
(oracle/ref_shim_rtr_serial.c): the threaded build reads its partial sums of log w - w before
joining the threads, so its nu depends on thread timing."""
import numpy as np
import pytest

from util import small_problem, relerr

pytestmark = pytest.mark.gpu

JONES_TOL = 1e-5

CASES = [
    ("rtr", 4, dict(N=10, M=3, tilesz=10, seed=71), dict(max_iter=3)),
    ("rtr-hybrid", 4, dict(N=12, M=4, tilesz=10, seed=72, nchunk=[1, 2, 1, 5]), dict(max_iter=2)),
    ("rtr-uneven", 4, dict(N=9, M=3, tilesz=10, seed=73, nchunk=[3, 1, 4]), dict(max_iter=2)),
    ("rtr-flags", 4, dict(N=10, M=2, tilesz=10, seed=74, flag_frac=0.3, uvcut_frac=0.02),
     dict(max_iter=3)),
    ("rtr-nolbfgs", 4, dict(N=35, M=3, tilesz=6, seed=75), dict(max_iter=2, max_lbfgs=0)),
    # more than one time slice per baseline block and more than 32 stations per warp loop
    ("rtr-slices", 4, dict(N=40, M=2, tilesz=24, seed=76), dict(max_iter=2, max_lbfgs=0)),
    ("rrtr", 5, dict(N=10, M=3, tilesz=10, seed=77, outliers=0.02), dict(max_iter=3)),
    ("rrtr-hybrid", 5, dict(N=13, M=4, tilesz=20, seed=78, kmean=1.0, outliers=0.02,
                            nchunk=[1, 2, 1, 4]), dict(max_iter=2)),
    ("rrtr-62", 5, dict(N=62, M=3, tilesz=4, seed=79, outliers=0.02), dict(max_iter=2, max_lbfgs=4)),
    # more than 64 stations: Jones through device memory instead of the parameter block, several
    # baseline ends per 16-lane group
    ("rtr-70", 4, dict(N=70, M=2, tilesz=2, seed=82), dict(max_iter=2, max_emiter=2, max_lbfgs=2)),
    ("rrtr-70", 5, dict(N=70, M=2, tilesz=2, seed=83, outliers=0.02),
     dict(max_iter=2, max_emiter=2, max_lbfgs=0)),
    ("nsd", 6, dict(N=10, M=3, tilesz=10, seed=80, outliers=0.02), dict(max_iter=3)),
    ("nsd-hybrid", 6, dict(N=11, M=3, tilesz=12, seed=81, outliers=0.02, nchunk=[2, 1, 3]),
     dict(max_iter=2)),
    # 62 stations, 13 slots: the condensation's last time slice is short (7 slices of 2 and 1 on 132
    # or 114 SMs), as at C3rtr (9 slices of 14 and 8)
    ("rtr-62-ragged", 4, dict(N=62, M=2, tilesz=13, seed=84), dict(max_iter=2, max_lbfgs=4)),
    ("rrtr-62-ragged", 5, dict(N=62, M=2, tilesz=13, seed=85, outliers=0.02),
     dict(max_iter=2, max_lbfgs=4)),
    # hybrid: 26 slots in one chunk and two chunks of 13, all split with a short last slice
    ("rrtr-62-hybrid-ragged", 5, dict(N=62, M=2, tilesz=26, seed=86, outliers=0.02, nchunk=[1, 2]),
     dict(max_iter=2, max_lbfgs=0)),
]


@pytest.mark.parametrize("name,mode,prob,args", CASES, ids=[c[0] for c in CASES])
def test_sagefit_rtr_modes(api, ref, refser, name, mode, prob, args):
    b = small_problem(**prob)
    pr = b.pr
    kw = dict(max_emiter=3, max_lbfgs=6, lbfgs_m=7, randomize=0, solver_mode=mode)
    kw.update(args)
    out = []
    for lib in (ref if mode == 4 else refser, api):
        x = pr.x.copy()
        pp = pr.pp0.copy()
        r = lib.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(),
                                     b.sky, pr.coh, pp, **kw)
        out.append((r, x, pp))
    (rr, xr, ppr), (rg, xg, ppg) = out
    assert rr[0] == rg[0]
    assert abs(rr[1] - rg[1]) < 1e-9                    # mean nu
    assert abs(rr[2] - rg[2]) <= 1e-10 * rr[2]          # res_0
    assert relerr(ppg, ppr) < JONES_TOL, (name, relerr(ppg, ppr))
    assert relerr(xg, xr) < 1e-5 * max(1.0, np.max(np.abs(pr.x)) / np.max(np.abs(xr)))
    assert abs(rr[3] - rg[3]) <= 1e-5 * rr[3]           # res_1
    assert rg[3] <= rg[2]   # (the robust solvers may discard every visit, DESIGN.md 9b)


# At the exact solution the condensed tensors give the cost as c0 - Re(...), which cancels completely on
# noise-free data, so RSD + RTR (mode 4) may take steps on rounding noise: on one H100 this problem
# moves by 9.8e-11, the robust modes not at all.  The kernels' arithmetic run on the CPU moves other
# seeds of this problem by up to 6e-9 (DESIGN.md 5.3), so a change of rounding order in the kernels
# can call for another look at this bound.
@pytest.mark.parametrize("mode", [4, 5, 6])
def test_sagefit_rtr_at_the_solution(api, ref, refser, mode):
    """Noise-free data and the true Jones as the starting point (the twin of the LM family's
    test_sagefit_at_the_solution_stops_like_the_reference): the reference returns the Jones
    unchanged, the product within 1e-9"""
    b = small_problem(N=8, M=3, tilesz=6, seed=61, noise_rel=0.0, flag_frac=0.0, uvcut_frac=0.0)
    pr = b.pr
    out = []
    for lib in (ref if mode == 4 else refser, api):
        x = pr.x.copy()
        pp = pr.jones_true.copy()
        r = lib.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, b.fresh_barr(),
                                     b.sky, pr.coh, pp, max_emiter=2, max_iter=3, max_lbfgs=0,
                                     lbfgs_m=5, solver_mode=mode, randomize=0)
        out.append((r, pp))
    (rr, ppr), (rg, ppg) = out
    assert np.max(np.abs(ppr - pr.jones_true)) < 1e-9
    assert np.max(np.abs(ppg - pr.jones_true)) < 1e-9, np.max(np.abs(ppg - pr.jones_true))
    assert rg[2] < 1e-12 and rr[2] < 1e-12
