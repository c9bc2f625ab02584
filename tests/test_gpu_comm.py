"""Multi-GPU gather of the surfel deltas through the C ABI (dsm_comm_init / dsm_gather_deltas, csrc/dsm_comm.cu):
the payload the root receives from every rank must be byte-identical to gather.pack_payload() of what that rank's
dsm_batch_download returns.  One rank runs anywhere; the two-rank test needs two GPUs (gpurun --gpus 2)."""
import os

import numpy as np
import pytest

from densesurfelmapping_b200 import gather, synth
from densesurfelmapping_b200.elements import SURFEL_DTYPE

pytestmark = pytest.mark.gpu

CAM = synth.Camera(132, 100, 60.0, 60.0, 65.5, 49.5, 0.5, 30.0)
B = 3


def _run_batch(capi, device, rank):
    """Two passes on one context: the first seeds every frame's pool, the second (the one gathered) fuses + initialises."""
    ctx = capi.Context(CAM, max_batch=B, max_local_surfels=4096, device=device)
    frames = [synth.make_frame(CAM, 40 * rank + i, synth.pose_stream(i)) for i in range(B)]
    g, d = np.stack([f[0] for f in frames]), np.stack([f[1] for f in frames])
    p = np.stack([synth.pose_stream(i) for i in range(B)])
    _, pools = ctx.fuse_batch([0] * B, g, d, p, np.zeros(0, SURFEL_DTYPE), np.zeros(B + 1, np.int32))
    ofs = np.concatenate([[0], np.cumsum([len(x) for x in pools])]).astype(np.int32)
    ctx.batch_upload([1] * B, g, d, p, np.concatenate(pools), ofs)
    ctx.batch_run()
    local, news = ctx.batch_download()
    return ctx, gather.pack_payload(news, local, ofs)


def _single_rank_gather():
    from densesurfelmapping_b200 import capi
    ctx, want = _run_batch(capi, 0, 0)
    ctx.comm_init(capi.comm_unique_id(), 0, 1)
    for _ in range(2):  # twice: the staging buffers are reused
        ctx.gather_deltas(0)
        ctx.gather_wait()
        got = ctx.gathered_payload(0)
        assert got.tobytes() == want.tobytes()
    news, pool, ofs = gather.unpack_payload(got)
    assert len(news) == B and sum(len(a) for a in news) > 0 and len(pool) == ofs[-1] > 0
    ctx.close()


def test_single_rank_gather_equals_batch_download():
    """Peer transport: the pack kernel writes into the context's own slot."""
    _single_rank_gather()


def test_single_rank_nccl_gather_equals_batch_download(monkeypatch):
    """NCCL transport: the same pack kernel writes into the send buffer; the root copies its own payload into the receive
    buffer."""
    monkeypatch.setenv("DSM_GATHER_NCCL", "1")  # read by dsm_comm_init
    _single_rank_gather()


def _worker(rank, world, uid_q, res_q, transport="peer"):
    # no torch in these processes: the library then loads the system NCCL, as in a plain C++ host process
    if transport == "nccl":
        os.environ["DSM_GATHER_NCCL"] = "1"
    from densesurfelmapping_b200 import capi
    if rank == 0:
        uid = capi.comm_unique_id()
        for _ in range(world - 1):
            uid_q.put(uid)
    else:
        uid = uid_q.get(timeout=60)
    ctx, want = _run_batch(capi, rank, rank)
    ctx.comm_init(uid, rank, world)
    for _ in range(3):  # three gathers in a row: the slots / staging buffers are reused, the credits advance
        ctx.gather_deltas(0)
    ctx.gather_wait()
    if rank == 0:
        res_q.put(("root", [ctx.gathered_payload(r).tobytes() for r in range(world)]))
    res_q.put((rank, want.tobytes()))
    ctx.close()


def _gpu_count():
    import subprocess
    try:
        return len([l for l in subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=60).stdout.splitlines() if l.startswith("GPU ")])
    except Exception:
        return 0


@pytest.mark.parametrize("transport", ["peer", "nccl"])
def test_two_rank_gather(transport):
    """peer: one-sided writes into the root's CUDA-IPC-mapped slots over NVLink; nccl: counts + grouped send/recv."""
    # (torch is deliberately not imported here: this process may already hold the system NCCL from the single-rank test,
    # and a PyTorch that loads after it would bind to that one instead of its own -- INTEGRATION.md, "NCCL in a PyTorch process")
    if _gpu_count() < 2:
        pytest.skip("needs two GPUs (run with gpurun --gpus 2)")
    import multiprocessing as mp
    mpc = mp.get_context("spawn")
    uid_q, res_q = mpc.Queue(), mpc.Queue()
    procs = [mpc.Process(target=_worker, args=(r, 2, uid_q, res_q, transport)) for r in range(2)]
    [p.start() for p in procs]
    got = dict(res_q.get(timeout=180) for _ in range(3))
    [p.join(60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    assert got["root"][0] == got[0] and got["root"][1] == got[1] and got[0] != got[1]
