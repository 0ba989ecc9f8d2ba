"""GPU: the LM cluster passes directly.  k_cluster_pass_lin<5, false / true>, k_cluster_pass_split and
the tile k_cluster_pass (kernels_stream.cu) through db_cluster_pass, the one entry every LM, OS-LM,
robust LM and RTR visit uses (hook dirac_b200_cluster_pass_eval), and k_cluster_rowmap (kernels_line.cu)
through db_cluster_hidden (hook dirac_b200_cluster_hidden_eval), against util.cluster_pass_ref /
cluster_rowmap_ref, the plain per-row float64 restatements that tests/test_cpu_refs.py pins to the
compiled reference and to the hidden-data identities.

Cases (util.CP_CASES; N stations, T timeslots, nchunk of the clusters):
  n2         N 2, T 3: one baseline, 255 idle lanes per half of the linear-mapped CTA
  n7h        N 7, T 5, nchunk [1, 2, 3]: the case the CPU pin compares with the reference
  n23, n24   N 23 / 24, T 5, nchunk [1, 2, 3]: one ragged baseline group (253) versus two (the second
             of 20); chunks with t0 > 0, uneven chunks
  n9e        N 9, T 3, nchunk [1, 4]: an empty last chunk (db_cluster_pass returns before any launch)
  n9r        N 9, T 64, rows per CTA forced to 5 and 32: the staging ring wraps, two slices of 32 rows,
             flag bit 31
  n62        N 62, T 120: the default slicing at a C2 / C3 sized chunk
  n512       N 512, T 2: the C4 station count, 8N = 4096 station sums in shared memory
  n639, n640 the largest array the linear-mapped kernel takes (204 776 of 204 800 bytes of shared
             memory), and the smallest where k_cluster_pass_split and the tile kernel take every pass
Every case has random flag-1 and uv-cut rows with non-zero data, one fully flagged station (N > 2)
and one fully flagged timeslot.  Each (cluster, chunk) runs the passes of util.CP_RUNS.  The file
reads nothing of the reference."""
import numpy as np
import pytest

from sagecal_b200 import lib as blib
from sagecal_b200.dirac_api import SkyModel, make_barr
from util import (CP_CASES, CP_RUNS, cluster_case, cluster_pass_ref, cluster_rowmap_ref,
                  cp_expected_kernel, cp_ref_args, cp_run_applies)

pytestmark = pytest.mark.gpu

_cases = {}

#: kinds of db_prof_begin a cluster pass counts under (gradient-carrying; ADD / SUB / cost-only)
PASS_KINDS = (2, 8)


def _case(name):
    if name not in _cases:
        _cases[name] = cluster_case(name)
    return _cases[name]


def _problem(api, c):
    pr = c["pr"]
    return blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, make_barr(pr.sta1, pr.sta2, pr.flag),
                              SkyModel(pr.clusters, pr.N), pr.coh, pr.x)


def _passes(api):
    return sum(api.kernel_count(kd) for kd in PASS_KINDS)


def _ratio(err, bound):
    err = np.asarray(err, dtype=np.float64)
    return float(np.max(np.where(err == 0, 0.0, err / np.maximum(bound, 1e-300)), initial=0.0))


def _call(dp, k, ck, a):
    return dp.cluster_pass(k, ck, a["mode"], a["pblk"], a["x"], write_out=a["write_out"],
                           with_jte=a["with_jte"], form_hidden=a["form_hidden"], beta=a["beta"],
                           pblk_old=a["pblk_old"], wt=a["wt"], out_init=a["out_init"],
                           inplace=a["inplace"])


#: runs repeated to check that the same call gives the same bits
REPEAT = ("init", "trial_wt", "sub_rec8")


@pytest.mark.parametrize("name,cp_rows", [("n2", 0), ("n7h", 0), ("n23", 0), ("n24", 0), ("n9e", 0),
                                          ("n9r", 5), ("n9r", 32), ("n62", 0), ("n512", 0),
                                          ("n639", 0), ("n640", 0)])
def test_cluster_passes_match_restatement(api, name, cp_rows):
    """every pass of util.CP_RUNS on every (cluster, chunk): the kernel the dispatch picks, one launch
    (none for an empty chunk), the output within its bound on the chunk's rows and bit-equal to the
    output vector's previous content elsewhere (everywhere without write_out), bit-equal to the input
    on flagged rows at beta 1, the cost and J^T e within their bounds, J^T e exactly 0 at the fully
    flagged station.  Repeated calls give the same output and cost bits; J^T e too where one baseline
    group carries the linear-mapped pass.  With several groups k_cluster_pass_lin adds the group
    totals to J^T e with atomicAdd, and the split kernel adds every CTA's station sums so, in an order
    that varies: there J^T e is held to its bound only."""
    c = _case(name)
    N = c["N"]
    fs = N // 2 if N > 2 else None
    worst = dict(out=0.0, cost=0.0, jte=0.0)
    kernels = set()
    api.set_option("cp_rows", cp_rows)
    try:
        with _problem(api, c) as dp:
            for k in range(c["M"]):
                for ck in range(c["nchunk"][k]):
                    for run, kw in CP_RUNS:
                        if not cp_run_applies(c, run, kw):
                            continue
                        a = cp_ref_args(c, k, ck, kw)
                        want_kernel = cp_expected_kernel(c, k, ck, kw)
                        n0 = _passes(api)
                        got = _call(dp, k, ck, a)
                        where = (k, ck, run)
                        assert got["kernel"] == want_kernel, where
                        assert _passes(api) - n0 == (0 if want_kernel == "none" else 1), where
                        kernels.add(got["kernel"])
                        r = cluster_pass_ref(c, k, ck, **a)
                        err = np.abs(got["out"] - r["out"])
                        assert (err <= r["out_bound"]).all(), (where, _ratio(err, r["out_bound"]))
                        worst["out"] = max(worst["out"], _ratio(err, r["out_bound"]))
                        r0, r1 = r["rows"]
                        if a["write_out"] and a["beta"] == 1.0:
                            fl = np.zeros(len(c["flag"]), dtype=bool)
                            fl[r0:r1] = c["flag"][r0:r1] != 0
                            fl8 = np.repeat(fl, 8)
                            assert np.array_equal(got["out"][fl8], a["x"][fl8]), where
                        if a["mode"] in (0, 1, 4):
                            e = abs(got["cost"] - r["cost"])
                            assert e <= r["cost_bound"], (where, got["cost"], r["cost"])
                            worst["cost"] = max(worst["cost"], _ratio(e, r["cost_bound"]))
                        else:
                            assert got["cost"] == 0.0
                        err = np.abs(got["jte"] - r["jte"])
                        assert (err <= r["jte_bound"]).all(), (where, _ratio(err, r["jte_bound"]))
                        worst["jte"] = max(worst["jte"], _ratio(err, r["jte_bound"]))
                        if fs is not None:
                            assert not got["jte"][8 * fs:8 * fs + 8].any(), where
                        if run in REPEAT:
                            again = _call(dp, k, ck, a)
                            assert np.array_equal(again["out"], got["out"]), where
                            assert again["cost"] == got["cost"], where
                            if got["kernel"] == "lin_grad" and c["Nbase"] <= 256:
                                assert np.array_equal(again["jte"], got["jte"]), where
                            else:
                                assert (np.abs(again["jte"] - r["jte"]) <= r["jte_bound"]).all()
    finally:
        api.set_option("cp_rows", 0)
    lin = N <= 639
    assert kernels - {"none"} == ({"lin", "lin_grad", "split", "tile"} if lin else {"split", "tile"})
    print("cluster passes %s (rows per CTA %s): kernels %s; largest error / bound: output %.3g, "
          "cost %.3g, J^T e %.3g" % (name, cp_rows or "default", sorted(kernels), worst["out"],
                                     worst["cost"], worst["jte"]))


@pytest.mark.parametrize("name", ["n7h", "n23", "n24", "n9e"])
def test_cluster_rowmap_matches_restatement(api, name):
    """db_cluster_hidden on every cluster, sign +1 (hidden data beta r + f) and -1 (residual d - f
    + (1-beta) r, read from and written to the same vector r when beta != 1) at beta 1 and 1/8: within
    the bound, bit-equal to the input on flagged rows at beta 1, one launch"""
    c = _case(name)
    r, dh = c["y"], c["x"]
    fl8 = np.repeat(c["flag"] != 0, 8)
    worst = 0.0
    with _problem(api, c) as dp:
        for k in range(c["M"]):
            for sign in (1, -1):
                for beta in (1.0, 0.125):
                    n0 = api.launch_count()
                    got = dp.cluster_hidden(k, sign, beta, c["P_old"], r, dh)
                    # uploads of r and dh, the pass, the download
                    assert api.launch_count() - n0 == 4
                    want, bound = cluster_rowmap_ref(c, k, sign, beta, c["P_old"], r, dh)
                    err = np.abs(got - want)
                    assert (err <= bound).all(), (k, sign, beta, _ratio(err, bound))
                    worst = max(worst, _ratio(err, bound))
                    if beta == 1.0:
                        assert np.array_equal(got[fl8], (r if sign > 0 else dh)[fl8])
    print("row map %s: largest error / bound %.3g" % (name, worst))


def test_cluster_pass_refusals(api):
    """every refusal returns -1 before any device work (no launch, nothing written) and leaves the
    resident problem as it was: the same valid call gives the same bits before and after"""
    for name in ("n24", "n640"):
        c = _case(name)
        with _problem(api, c) as dp:
            ok = cp_ref_args(c, 1 if c["M"] > 1 else 0, 0, dict(mode=1, with_jte=True, wt=True))
            first = _call(dp, 1 if c["M"] > 1 else 0, 0, ok)
            assert first["kernel"] == "split"
            base = cp_ref_args(c, 0, 0, dict(mode=1, old=True))
            bad = [(c["M"], 0, {}), (-1, 0, {}), (0, c["nchunk"][0], {}), (0, -1, {}),
                   (0, 0, dict(mode=5)), (0, 0, dict(mode=-1)), (0, 0, dict(mode=4)),
                   (0, 0, dict(mode=2, with_jte=True)), (0, 0, dict(mode=3, with_jte=True)),
                   (0, 0, dict(form_hidden=True, mode=0)), (0, 0, dict(form_hidden=True, mode=2)),
                   (0, 0, dict(form_hidden=True, wt=c["wt"])),
                   (0, 0, dict(form_hidden=True, pblk_old=None)),
                   (0, 0, dict(mode=3, beta=0.5, pblk_old=None))]
            if name == "n640":
                bad.append((0, 0, dict(form_hidden=True)))   # the linear-mapped kernel does not fit
            n0, p0 = api.launch_count(), _passes(api)
            for k, ck, over in bad:
                a = dict(base, **over)
                got = _call(dp, k, ck, a)
                assert got["kernel"] is None, (name, k, ck, over)
                assert np.isnan(got["out"]).all() and np.isnan(got["jte"]).all()
                assert np.isnan(got["cost"])
            assert dp.cluster_hidden(c["M"], 1, 1.0, c["P"], c["y"], c["x"]) is None
            assert dp.cluster_hidden(0, 0, 1.0, c["P"], c["y"], c["x"]) is None
            assert (api.launch_count(), _passes(api)) == (n0, p0)
            after = _call(dp, 1 if c["M"] > 1 else 0, 0, ok)
            assert np.array_equal(after["out"], first["out"]) and after["cost"] == first["cost"]
