"""Multi-GPU (>= 2 H100s on one box): view-sharded inference through the real engine
with the single NCCL all_gather equals the single-GPU result bit for bit."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    import torch.distributed as dist
    from casmvsnet_pl_b200 import ABN, synth
    from casmvsnet_pl_b200.dist import sharded_depth_inference
    from casmvsnet_pl_b200.models.mvsnet import CascadeMVSNet
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    torch.set_grad_enabled(False)            # inference, like eval.py:219
    dist.init_process_group("nccl", rank=rank, world_size=world,
                            device_id=torch.device("cuda", rank))
    try:
        torch.manual_seed(0)
        m = CascadeMVSNet(norm_act=ABN, precision="tf32")
        synth.randomize_model_(m, 0)
        m = m.eval().cuda()
        imgs, pm, dmin, dint = synth.make_inputs(B=3, V=3, W=320, H=256, seed=4)
        imgs, pm = imgs.cuda(), pm.cuda()
        # per-view engine call so that sharded and unsharded runs use identical cuDNN shapes
        def engine(i, p, a, b):
            outs = [m(i[k:k + 1], p[k:k + 1], a, b) for k in range(i.shape[0])]
            return {key: torch.cat([o[key] for o in outs], 0) for key in outs[0]}
        got = sharded_depth_inference(engine, imgs, pm, dmin, dint)
        want = engine(imgs, pm, dmin, dint)
        q.put((rank, bool(torch.equal(got["depth_0"], want["depth_0"])),
               bool(torch.equal(got["confidence_2"], want["confidence_2"]))))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_sharded_engine_equals_single_gpu():
    import torch.multiprocessing as mp
    world = 2
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(d and c for _, d, c in got)
