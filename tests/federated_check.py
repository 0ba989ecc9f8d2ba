"""Run under torch.distributed.run with 2 processes (tests/test_gpu_federated_interval.py launches it):
one federated stochastic interval per rank, each rank on its own measurement set (interval `rank` of
the shared problem), exchanging through the gloo callback (both ranks on one device) or the library's
NCCL communicator (one device per rank).  Each rank saves its outputs to <out>/rank<r>.npz; the
pytest process compares them with a one-process emulation of the slaves and the master."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from sagecal_b200 import lib as blib, dist as sdist  # noqa: E402
from test_gpu_federated_interval import fed_setup, run_call  # noqa: E402


def main():
    backend, out = sys.argv[1], sys.argv[2]
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    api = blib.load()
    if backend == "gloo":
        torch.cuda.set_device(0)
        dist.init_process_group("gloo")
        cb = sdist.make_allreduce("cuda")
    else:
        torch.cuda.set_device(rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", rank))
        sdist.init_nccl(api, rank, world)
        cb = None
    b, sky, ivls, setup = fed_setup(api, world)
    got = run_call(api, b, sky, ivls[rank], setup, rank=rank, world=world, allreduce=cb)
    np.savez(os.path.join(out, "rank%d.npz" % rank), *got)
    dist.barrier()
    if backend != "gloo":
        api.lib.dirac_b200_nccl_finalize()
    dist.destroy_process_group()
    print("FEDERATED_CHECK OK rank %d" % rank)


if __name__ == "__main__":
    main()
