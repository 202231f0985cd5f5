"""D1 on hardware: gvd_b200.train.Trainer on 2 GPUs over NCCL — one ncclAllReduce of the flat gradient buffer per step — against the
single-process two-shard reference (tests/test_dist_gloo.py).  Needs >= 2 GPUs; skipped on a 1-GPU box."""
import pytest
import torch
import torch.multiprocessing as mp

from test_dist_gloo import _free_port, _single_process_two_shard_trainer, _trainer_worker

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_nccl_trainer_matches_single_process():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_trainer_worker, args=(r, world, port, q, "nccl", "cuda")) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted(q.get(timeout=600) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    ref, norms = _single_process_two_shard_trainer()
    stride = max(1, ref.numel // 257)
    for rank, n, wn, sample, calls, numel in results:
        assert calls == [numel, numel]
        assert all(abs(a - b) <= 2e-4 * b for a, b in zip(n, norms))
        assert abs(wn - ref.flat_w.double().norm().item()) <= 1e-5 * wn
        assert torch.allclose(torch.tensor(sample), ref.flat_w[::stride], rtol=0, atol=2 * 5e-4 * 2)
    assert results[0][1:4] == results[1][1:4]
