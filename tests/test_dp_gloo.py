"""world_size-2 `gloo` test of the data-parallel host logic (no GPU): the flat gradient arena is exchanged with ONE
all-reduce and averaged by 1/world inside the optimizer's grad_scale, which must equal training on the concatenated
batch (train_text_to_image_control_lora.py: DDP average of the ControlLoRA gradients, SURVEY.md §8e)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from controllora_b200.arena import ParamArena
    import controllora_b200 as cb
    from controllora_b200.configs import NAMED

    torch.manual_seed(0)                       # identical initial parameters on every rank (accelerate set_seed)
    cl = cb.ControlLoRA.from_config(NAMED["diffusiondb-canny-v2"])
    arena = ParamArena(list(cl.parameters()), torch.device("cpu"))
    # parameters were re-homed into the arena without changing identity or values
    assert sum(p.numel() for p in cl.parameters()) == arena.numel
    first = next(cl.parameters())
    assert first.data.data_ptr() == arena.flat_p.data_ptr()
    g = torch.Generator().manual_seed(100 + rank)
    local = torch.randn(arena.flat_g.shape, generator=g)
    arena.flat_g.copy_(local)
    arena.all_reduce()                         # ONE collective over the whole arena
    gathered = [torch.zeros_like(local) for _ in range(world)]
    dist.all_gather(gathered, local)
    want = sum(gathered)
    ok = torch.allclose(arena.flat_g, want, atol=1e-6)
    # the per-parameter grad views alias the arena
    off_ok = torch.equal(arena.grad_of(first).flatten(), arena.flat_g[: first.numel()])
    scale_ok = abs(arena.grad_scale - 1.0 / world) < 1e-12
    q.put((rank, bool(ok), bool(off_ok), bool(scale_ok)))
    dist.destroy_process_group()


def test_flat_arena_allreduce_world2():
    world = 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(r[0] for r in res) == [0, 1]
    assert all(r[1] and r[2] and r[3] for r in res), res


def _seed_worker(rank, world, port, q):
    """Ranks seeded DIFFERENTLY: the arena must broadcast rank 0's parameters (accelerate/DDP does, train_...:513)."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from controllora_b200.arena import ParamArena
    import controllora_b200 as cb
    from controllora_b200.configs import NAMED

    torch.manual_seed(1234 + rank)
    cl = cb.ControlLoRA.from_config(NAMED["diffusiondb-canny-v2"])
    arena = ParamArena(list(cl.parameters()), torch.device("cpu"))
    gathered = [torch.zeros_like(arena.flat_p) for _ in range(world)]
    dist.all_gather(gathered, arena.flat_p)
    same = all(torch.equal(gathered[0], g) for g in gathered)
    nonzero = float(arena.flat_p.abs().sum()) > 0
    # the parameters still alias the arena after the broadcast
    alias = next(cl.parameters()).data.data_ptr() == arena.flat_p.data_ptr()
    q.put((rank, bool(same), bool(nonzero), bool(alias)))
    dist.destroy_process_group()


def test_arena_broadcasts_initial_parameters_world2():
    world = 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_seed_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert all(r[1] and r[2] and r[3] for r in res), res


def _trainer_worker(rank, world, port, q):
    """Real Trainer forward/backward on rank-local half batches (host-logic mode: kernels replaced by their torch restatements,
    tests/emu_ops.py) with ONE all-reduce of the arena; reference = a world-1 Trainer on the concatenated batch in the same process."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), CLB_EMU="1")
    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    solo = [dist.new_group([r]) for r in range(world)][rank]          # a 1-rank group: world == 1 inside an initialised job
    from tests import check_unet                                      # installs the emulation (tests/_device.py)
    from controllora_b200.trainer import Trainer

    def build(pg):
        _, munet, _, mcl = check_unet.build_pair("v1_stacked")        # v1 processors + a stacked pre-LoRA: > 16 queued reductions
        return Trainer(munet, mcl, lr=1e-3, process_group=pg)

    B, HW = 4, 16
    g = torch.Generator().manual_seed(5)
    full = [torch.randn(B, 4, HW, HW, generator=g), torch.randint(0, 1000, (B,), generator=g).float(),
            torch.randn(B, 77, 64, generator=g).to(torch.bfloat16), (torch.rand(B, 3, HW * 8, HW * 8, generator=g) * 2 - 1),
            torch.randn(B, 4, HW, HW, generator=g)]
    half = [v[rank * (B // world):(rank + 1) * (B // world)].contiguous() for v in full]
    tr = build(None)
    assert tr.world == world
    tr._forward_backward(*half)
    tr.arena.all_reduce()
    got = (tr.flat_g[:tr.numel] * tr.arena.grad_scale).clone()
    # two full optimizer steps: replicas must stay bit-identical
    tr.flat_g.zero_()
    for _ in range(2):
        tr.step(*half)
    gathered = [torch.empty_like(tr.flat_p) for _ in range(world)]
    dist.all_gather(gathered, tr.flat_p)
    in_sync = all(torch.equal(gathered[0], t) for t in gathered[1:])
    big = build(solo)
    assert big.world == 1
    big._forward_backward(*full)
    want = big.flat_g[:big.numel].clone()
    q.put((rank, float((got - want).norm() / want.norm()), in_sync))
    dist.barrier()
    dist.destroy_process_group()


def test_trainer_gradient_exchange_world2():
    """SURVEY 8(e): DP on half batches with one all-reduce == single process on the concatenated batch."""
    world = 2
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_trainer_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=120)
    for rank, err, in_sync in res:
        # the sharp check: the replicas stay bit-identical over optimizer steps
        assert in_sync, res
        # against the concatenated batch only a loose bound is meaningful on the CPU: the BLAS behind the torch restatements is not
        # batch-invariant at the 1e-7 level and bf16 rounding decorrelates after a few layers (two runs of the same samples at
        # different batch sizes differ like two independent bf16 pipelines, ~1.5e-2).  The real kernels are batch-invariant: the
        # 2-GPU NCCL test (tests/test_multigpu_nccl.py) holds 2e-3.
        assert err < 5e-2, res
