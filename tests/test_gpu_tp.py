"""Tensor-parallel VQuantLinear on real GPUs over NCCL (needs >= 2 GPUs; skipped otherwise)."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import sys
        here = os.path.dirname(os.path.abspath(__file__))
        for p in (os.path.dirname(here), os.path.join(os.path.dirname(here), "oracle"), here):
            sys.path.insert(0, p)
        import vptq_oracle as vo
        from _gpu import make_module, x_to_t
        from vptq_b200 import tp
        errs = []
        for kw in (dict(in_features=1024, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256),
                   dict(in_features=1024 + 128, out_features=512, vector_len=8, num_centroids=4096, num_res_centroids=256,
                        outlier_size=128, outlier_vector_len=4, num_outlier_centroids=4096, bias=True)):
            L = vo.make_layer(seed=5, **kw)
            full = make_module(L, f"cuda:{rank}")
            for mode in ("all_reduce", "all_gather"):
                m = tp.shard_module(full, rank, world, mode=mode)
                for tokens in (1, 2, 40):
                    x_np = vo.make_x(tokens, L.in_features, L.dtype, seed=tokens)
                    y = m(x_to_t(x_np, L, f"cuda:{rank}"))
                    torch.cuda.synchronize()
                    y_star = vo.quant_gemm(x_np, L)
                    errs.append(float(np.abs(y.float().cpu().numpy() - y_star).max() / np.abs(y_star).max()))
        q.put((rank, max(errs)))
    finally:
        dist.destroy_process_group()


def test_tp_two_gpus_nccl():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, err in res:
        assert err <= 1e-3, (rank, err)


def _worker_p2p(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        import sys
        here = os.path.dirname(os.path.abspath(__file__))
        for p in (os.path.dirname(here), os.path.join(os.path.dirname(here), "oracle"), here):
            sys.path.insert(0, p)
        import vptq_oracle as vo
        from _gpu import make_module, x_to_t
        from vptq_b200 import native, tp
        # two chained layers: A (1024 -> 2048) then B (2048 -> 1024); x of B = exchanged output of A
        LA = vo.make_layer(in_features=1024, out_features=2048, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=41)
        LB = vo.make_layer(in_features=2048, out_features=1024, vector_len=8, num_centroids=4096, num_res_centroids=256, seed=42)
        shards = []
        for L in (LA, LB):
            full = make_module(L, f"cuda:{rank}")
            sh = tp.shard_module(full, rank, world).shard
            sh(torch.zeros(0, L.in_features, device=dev, dtype=torch.float16))     # builds the descriptor
            shards.append(sh)
        arena = tp.PeerArena(1 << 20, dev)
        yA, offA = arena.alloc((1, 2048), torch.float16)
        yB, offB = arena.alloc((1, 1024), torch.float16)
        flags, off_flags = arena.alloc((2, world), torch.int32)
        epoch = torch.zeros(2, dtype=torch.int32, device=dev)
        done = torch.zeros(2, dtype=torch.int32, device=dev)
        error = torch.zeros(1, dtype=torch.int32, device=dev)
        locA, locB = 2048 // world, 1024 // world
        exA = tp.make_exchange(arena, slot=0, wait_slot=-1, y_offsets=[offA], slice_bytes=[rank * locA * 2],
                               flags_offset=off_flags, epoch=epoch, done=done, error=error, num_slots=2)
        exB = tp.make_exchange(arena, slot=1, wait_slot=0, y_offsets=[offB], slice_bytes=[rank * locB * 2],
                               flags_offset=off_flags, epoch=epoch, done=done, error=error, num_slots=2)
        fA = native.FusedGemvTP([shards[0]._desc_cache[0]], [yA[:, rank * locA:(rank + 1) * locA]], exA)
        fB = native.FusedGemvTP([shards[1]._desc_cache[0]], [yB[:, rank * locB:(rank + 1) * locB]], exB)
        errs = []
        for it in range(4):                      # repeated tokens: epochs advance, buffers are reused
            x_np = vo.make_x(1, 1024, "fp16", seed=100 + it)
            x = x_to_t(x_np, LA, f"cuda:{rank}")
            fA(x)
            fB(yA)
            torch.cuda.synchronize()
            dist.barrier()
            torch.cuda.synchronize()
            a_star = vo.quant_gemm(x_np, LA)
            a_got = yA.cpu().numpy()                                     # what layer B actually consumed
            b_star = vo.quant_gemm(a_got, LB)
            errs.append(float(np.abs(a_got.astype(np.float32) - a_star).max() / np.abs(a_star).max()))
            errs.append(float(np.abs(yB.float().cpu().numpy() - b_star).max() / np.abs(b_star).max()))
        # ---- the tagged wire format (8-byte words {2 values, tag}: no flags, no fences): both layers on the list
        # kernel, C reads the tagged buffer A wrote, 5 tokens so that tags advance and buffers are reused ----
        LC = vo.make_layer(in_features=2048, out_features=1024, vector_len=8, num_centroids=65536, num_res_centroids=256, seed=43)
        shC = tp.shard_module(make_module(LC, f"cuda:{rank}"), rank, world).shard
        shC(torch.zeros(0, LC.in_features, device=dev, dtype=torch.float16))
        tA, toffA = arena.alloc((1, 2048 * 4), torch.uint8)
        tC, toffC = arena.alloc((1, 1024 * 4), torch.uint8)
        pA = torch.zeros(1, 2048, device=dev, dtype=torch.float16)
        pC = torch.zeros(1, 1024, device=dev, dtype=torch.float16)
        epoch2 = torch.zeros(2, dtype=torch.int32, device=dev)
        done2 = torch.zeros(2, dtype=torch.int32, device=dev)
        kw = dict(flags_offset=off_flags, epoch=epoch2, done=done2, error=error, fmt=native.TP_TAGGED, num_slots=2)
        exA2 = tp.make_exchange(arena, slot=0, wait_slot=-1, y_offsets=[toffA], slice_bytes=[rank * locA * 4], **kw)
        exC2 = tp.make_exchange(arena, slot=1, wait_slot=0, y_offsets=[toffC], slice_bytes=[rank * locB * 4], **kw)
        gA = native.FusedGemvTP([shards[0]._desc_cache[0]], [pA[:, rank * locA:(rank + 1) * locA]], exA2)
        gC = native.FusedGemvTP([shC._desc_cache[0]], [pC[:, rank * locB:(rank + 1) * locB]], exC2)
        for it in range(5):
            x_np = vo.make_x(1, 1024, "fp16", seed=200 + it)
            gA(x_to_t(x_np, LA, f"cuda:{rank}"), native.FLAG_PDL)
            gC(tA, native.FLAG_PDL)
            # the chain's last activation has no tagged consumer: vptq_b200_tp_untag waits for every rank's words
            c_full = torch.zeros(1, 1024, device=dev, dtype=torch.float16)
            native.tp_untag(tC, c_full, exC2)
            torch.cuda.synchronize()
            c_early = c_full.float().cpu().numpy()
            dist.barrier()
            torch.cuda.synchronize()
            a_got = tp.untag(tA, torch.float16).cpu().numpy()
            c_got = tp.untag(tC, torch.float16).float().cpu().numpy()
            assert np.array_equal(c_early, c_got)
            a_star = vo.quant_gemm(x_np, LA)
            c_star = vo.quant_gemm(a_got, LC)
            errs.append(float(np.abs(a_got.astype(np.float32) - a_star).max() / np.abs(a_star).max()))
            errs.append(float(np.abs(c_got - c_star).max() / np.abs(c_star).max()))
            # the plain local slices the kernels also leave behind
            sl = slice(rank * locB, (rank + 1) * locB)
            assert torch.equal(pC[:, sl].cpu(), torch.from_numpy(c_got[:, sl]).half())
        q.put((rank, errs, int(error.item())))
    finally:
        dist.destroy_process_group()


def test_tp_fused_p2p_exchange_two_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker_p2p, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, errs, flag in res:
        assert flag == 0, "a flag wait timed out"
        assert max(errs) <= 1e-3, (rank, [f"{e:.2e}" for e in errs])
