"""2-GPU NCCL test (pytest -m gpu; skipped on boxes with fewer than 2 GPUs): after the real fused backward on each rank's
half batch and ONE ncclAllReduce of the flat gradient arena, (all-reduced arena) x 1/world must equal the gradient of a
single-GPU run on the concatenated batch (SURVEY.md 8e / section 4(iv): "grad-equality vs single-GPU big-batch"; reference:
DDP's bucketed all-reduce behind accelerator.backward, train_text_to_image_control_lora.py:790)."""
import os
import socket

import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _build(dev, pg=None):
    import controllora_b200 as cb
    from controllora_b200.configs import wire_processors
    from controllora_b200.trainer import Trainer
    from controllora_b200.unet import synthetic_state_dict
    from tests.check_unet import TINY, TINY_LORA

    unet = cb.UNet2DConditionModel.from_state_dict(synthetic_state_dict(TINY, 0), dev, TINY)
    torch.manual_seed(3)
    kw = dict(TINY_LORA)
    kw.update(lora_control_version=2, lora_pre_conv_skipped=True, lora_key_states_skipped=True, lora_value_states_skipped=True)
    cl = cb.ControlLoRA(**kw)
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for n_, p_ in cl.named_parameters():
            if n_.endswith("up.weight"):
                p_.copy_(0.05 * torch.randn(p_.shape, generator=g))
    cl.to(dev)
    wire_processors(unet, cl)
    return Trainer(unet, cl, lr=1e-4, process_group=pg)


def _inputs(B, HW=16):
    g = torch.Generator().manual_seed(9)
    x = torch.randn(B, 4, HW, HW, generator=g)
    t = torch.randint(0, 1000, (B,), generator=g).float()
    e = torch.randn(B, 77, 64, generator=g).to(torch.bfloat16)
    guide = torch.rand(B, 3, HW * 8, HW * 8, generator=g) * 2 - 1
    tgt = torch.randn(B, 4, HW, HW, generator=g)
    return x, t, e, guide, tgt


def _worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    dev = torch.device("cuda", rank)
    tr = _build(dev)
    B = 4
    full = _inputs(B)
    half = [v[rank * (B // world):(rank + 1) * (B // world)].to(dev) for v in full]
    tr._forward_backward(*half)
    tr.arena.all_reduce()                # one all-reduce of the whole arena
    torch.cuda.synchronize()
    g = (tr.flat_g[:tr.numel] * tr.arena.grad_scale).detach().cpu()
    # graph-replayed steps (forward + backward captured; all-reduce, clip, AdamW behind each replay) on rank-local data: the
    # replicas must stay bit-identical and the device step counter must follow the host's
    tr.flat_g.zero_()
    tg = _build(dev)
    tg.cuda_graph, tg.graph_warmup = True, 2
    losses = []
    for it in range(5):
        losses.append(tg.step(*half))
    torch.cuda.synchronize()
    gathered = [torch.empty_like(tg.flat_p) for _ in range(world)]
    dist.all_gather(gathered, tg.flat_p)
    same = all(torch.equal(gathered[0], t) for t in gathered[1:])
    info = dict(same=bool(same), graph=tg._graph is not None, step_dev=int(tg.step_dev.item()), step_idx=tg.step_idx,
                finite=bool(torch.isfinite(torch.stack([l.float() for l in losses])).all()))
    if rank == 0:
        q.put(g)
        q.put(info)
    dist.barrier()
    dist.destroy_process_group()


def test_allreduced_arena_equals_single_gpu_big_batch():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    g_dp = q.get(timeout=300)
    info = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
    print("2-GPU whole-step graph:", info)
    assert info["same"] and info["graph"] and info["finite"] and info["step_dev"] == info["step_idx"] == 5
    tr = _build(torch.device("cuda", 0))
    tr._forward_backward(*[v.cuda() for v in _inputs(4)])
    torch.cuda.synchronize()
    g_one = tr.flat_g[:tr.numel].detach().cpu()
    err = float((g_dp - g_one).norm() / g_one.norm())
    print(f"2-GPU all-reduced arena vs single-GPU batch-4 gradient: rel {err:.3e}")
    assert err < 2e-3
