"""Run a function in `world` spawned processes that form one torch.distributed group, join them with a deadline and
leave none behind."""
import os
import socket
import time

import torch.multiprocessing as mp


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def run_group(fn, world, args, timeout=600):
    """fn(rank, world, port, *args) in `world` processes; raises (after killing the rest) if one fails or the deadline
    passes."""
    ctx = mp.start_processes(fn, args=(world, free_port()) + tuple(args), nprocs=world, join=False,
                             start_method="spawn")
    deadline = time.monotonic() + timeout
    try:
        while not ctx.join(timeout=2):
            if time.monotonic() > deadline:
                raise TimeoutError("the %d processes did not finish within %d s" % (world, timeout))
    finally:
        for p in ctx.processes:
            if p.is_alive():
                p.kill()
            p.join()


def init_group(rank, world, port, backend, **kw):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
