"""GPU, two processes: RemoteReader.distributed exchanges real CUDA IPC blobs, and each rank serves its own requests while
the other is idle (waiting in a barrier on the host).  On cuda:0 and cuda:1 with two GPUs, else both on cuda:0 (CUDA IPC
opens a handle in another process on the same device too).  Every returned row is the
owner's entry, rounded to f16 as the sharded path rounds it."""
import os
import socket
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu


def _entries(signs, dim):
    """The entry every sign is given: a function of the sign alone, so any rank knows every owner's rows."""
    s = signs.astype(np.float64)
    return (np.sin(s[:, None] * 0.001 + np.arange(dim)[None, :]) * 0.5).astype(np.float32)


def _rank_main(rank, world, port, result_dir, devices):
    import torch
    import torch.distributed as dist

    from persia_b200 import native as N
    from persia_b200 import shard as SH
    from persia_b200.worker import RemoteReader

    torch.cuda.set_device(devices[rank])
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    dev = torch.device("cuda", devices[rank])
    dim, n = 64, 5000
    signs = np.arange(1, n + 1, dtype=np.uint64)
    d_signs = torch.from_numpy(signs.view(np.int64)).to(dev)
    owner = SH.shard_of(d_signs, world).cpu().numpy()
    s = SH.EmbeddingShard(dim, 1 << 14, dev)
    s.set_optimizer(N.OPT_SGD, lr=0.1)
    mine = signs[owner == rank]
    s.set_entries(torch.from_numpy(mine.view(np.int64)).to(dev), torch.from_numpy(_entries(mine, dim)).to(dev))
    torch.cuda.synchronize()
    rd = RemoteReader.distributed(s)
    want = _entries(signs, dim).astype(np.float16)
    ok = True
    for turn in range(world):  # one rank serves, the other idles in the barrier
        if turn == rank:
            q = torch.from_numpy(np.concatenate([signs, [10 ** 9]]).astype(np.uint64).view(np.int64)).to(dev)
            out = rd.forward(q, n + 1, [0])
            torch.cuda.synchronize()
            got = out[0].cpu().numpy()
            ok = ok and bool((got[:n].view(np.uint16) == want.view(np.uint16)).all()) and not got[n].any()
        dist.barrier()
    ok = ok and s.counters()["wait_errors"] == 0
    rd.close()
    dist.barrier()  # every view closed before any table goes
    s.close()
    with open(os.path.join(result_dir, f"r{rank}"), "w") as f:
        f.write("ok" if ok else "bad")
    dist.destroy_process_group()


def test_two_processes_serve_alone(tmp_path):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import torch.multiprocessing as mp

    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        port = so.getsockname()[1]
    devices = [0, 1] if torch.cuda.device_count() >= 2 else [0, 0]
    mp.spawn(_rank_main, args=(2, port, str(tmp_path), devices), nprocs=2, join=True)
    assert [open(tmp_path / f"r{r}").read() for r in range(2)] == ["ok", "ok"]
