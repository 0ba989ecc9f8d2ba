"""Run under torchrun on >= 2 GPUs (tests/test_gpu_minibatch_stage.py launches it): the stochastic
LBFGS stage of sagefit (lbfgs_m < 0, robust solver_mode 2) alone (max_emiter=0) on a cluster-sharded
problem against the same stage on one GPU.  Sharded, each window's cost sums only the window's partial
models over the ranks and the gradient is summed over the parameters; the two runs differ by the order
of the sums only, so the Jones agree to 1e-9 and every rank holds bit-identical Jones."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sagecal_b200 import lib as blib, dist as sdist, synth  # noqa: E402
from sagecal_b200.dirac_api import SkyModel, make_barr, dptr  # noqa: E402


def main():
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    api = blib.load()
    stream = torch.cuda.Stream()
    api.set_stream(stream.cuda_stream)
    rep = {}
    with torch.cuda.stream(stream):
        # windows of ceil(16 * 15 / 2 * 11 / 5) = 264 rows cut timeslots of 120 rows
        pr = synth.make_problem(N=16, M=4 * world, tilesz=11, seed=101, kmean=1.0, outliers=0.02,
                                flag_frac=0.1)
        barr = make_barr(pr.sta1, pr.sta2, pr.flag)
        sky = SkyModel(pr.clusters, pr.N)
        rng = np.random.default_rng(102)
        p0 = pr.pp0 + 0.05 * rng.normal(0, 1, pr.pp0.shape)
        dp = blib.DeviceProblem(api, pr.N, pr.Nbase, pr.tilesz, barr, sky, pr.coh, pr.x)
        sp = sdist.ShardedProblem(api, pr, barr, rank, world)
        # one window's cost and gradient through the thin layer
        r0, nr = 264, 264
        c1, g1 = dp.cost_window(p0, r0, nr, 3.0), dp.grad_window(p0, r0, nr, 3.0)
        cs = api.lib.dirac_b200_cost_window(sp.h, dptr(p0), r0, nr, 3.0)
        gs = np.zeros_like(p0)
        api.lib.dirac_b200_grad_window(sp.h, dptr(p0), dptr(gs), r0, nr, 3.0)
        rep["window_cost"] = abs(cs - c1) / c1
        rep["window_grad"] = float(np.max(np.abs(gs - g1)) / np.max(np.abs(g1)))
        kw = dict(max_emiter=0, max_iter=0, max_lbfgs=10, lbfgs_m=-7, solver_mode=2)
        p1, ps = p0.copy(), p0.copy()
        r1 = dp.sagefit(p1, None, **kw)
        rs = sp.sagefit(ps, None, **kw)
        rep["stage_jones"] = float(np.max(np.abs(ps - p1)) / np.max(np.abs(p1)))
        rep["stage_moved"] = float(np.max(np.abs(p1 - p0)) / np.max(np.abs(p0)))
        rep["stage_res1"] = abs(rs[3] - r1[3]) / r1[3]
        sp.close()
        dp.close()
        t = torch.from_numpy(np.concatenate([ps, [rs[3]]])).cuda()
        t0 = t.clone()
        dist.broadcast(t0, 0)
        same = torch.tensor([1.0 if torch.equal(t, t0) else 0.0], device="cuda")
        dist.all_reduce(same, op=dist.ReduceOp.MIN)
        rep["identical_on_ranks"] = bool(same.item() > 0.5)
    rep["ok"] = bool(rep["window_cost"] < 1e-12 and rep["window_grad"] < 1e-11
                     and rep["stage_jones"] < 1e-9 and rep["stage_moved"] > 1e-6
                     and rep["stage_res1"] < 1e-9 and rep["identical_on_ranks"])
    if rank == 0:
        print(json.dumps(rep))
        print("MINIBATCH_STAGE_CHECK", "OK" if rep["ok"] else "FAIL")
    api.lib.dirac_b200_nccl_finalize()
    dist.destroy_process_group()
    sys.exit(0 if rep["ok"] else 1)


if __name__ == "__main__":
    main()
