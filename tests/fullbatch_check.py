"""Run under torch.distributed.run with 2 processes (tests/test_gpu_fullbatch.py launches it): one sharded
full-batch tile call per rank on the same tile, exchanging through the gloo callback (both ranks on one
device) or the library's NCCL communicator (one device per rank), then the same fit through the existing
sharded path (dirac_b200_create_shard, dirac_b200_precalculate, dirac_b200_sagefit).  Each rank saves its
outputs to <out>/rank<r>.npz; the pytest process compares them."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from sagecal_b200 import lib as blib, dist as sdist  # noqa: E402
from test_gpu_fullbatch import FREQS, emulate_rank, sharded_setup, tile  # noqa: E402


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
    b, sky, x, xo, kw = sharded_setup()
    got = tile(api, b, sky, x, xo, FREQS, b.pr.pp0, rank=rank, world=world, allreduce=cb, **kw)
    ep, ex, es = emulate_rank(api, rank, world, b, sky, x, kw)
    np.savez(os.path.join(out, "rank%d.npz" % rank), x=got["x"], xo=got["xo"], p=got["p"],
             flag=got["flag"], stats=np.array([got["nu"], got["r0"], got["r1"]]), emu_p=ep, emu_x=ex,
             emu_stats=es)
    dist.barrier()
    if backend != "gloo":
        api.lib.dirac_b200_nccl_finalize()
    dist.destroy_process_group()
    print("FULLBATCH_CHECK OK rank %d" % rank)


if __name__ == "__main__":
    main()
