"""TEST INFRASTRUCTURE ONLY: compares a product result with the compiled reference (its recorded
answers, oracle/refreplay.py)."""
import numpy as np

import refdirac


def check_sagefit(pr, barr, sky, pp_got, x_got, r0, r1, tol=1e-5, serial=False, **kw):
    """serial: against the reference build whose robust RTR / NSD solvers run their worker threads
    synchronously (the threaded build's nu update races, ref_shim_rtr_serial.c)"""
    ref = refdirac.recorded(serial)
    x = pr.x.copy()
    pp = pr.pp0.copy()
    args = dict(max_emiter=3, max_iter=5, max_lbfgs=10, lbfgs_m=7, solver_mode=1)
    args.update(kw)
    rv, nu, q0, q1 = ref.sagefit_visibilities(pr.u, pr.v, pr.w, x, pr.N, pr.Nbase, pr.tilesz, barr,
                                              sky, pr.coh, pp, **args)
    ej = np.max(np.abs(pp - pp_got)) / np.max(np.abs(pp))
    ex = np.max(np.abs(x - x_got)) / np.max(np.abs(pr.x))
    assert abs(q0 - r0) <= 1e-9 * q0, (q0, r0)
    assert ej < tol, "Jones differ from the reference by %g" % ej
    assert ex < tol, "residual differs from the reference by %g" % ex
    return ej, ex
