"""2-GPU check (a plain python script that spawns 2 ranks on a machine with 2 or more GPUs): data-parallel step == single-GPU step."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tiny-cuda-nn_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

CFG = json.load(open(os.path.join(ROOT, "tests", "golden", "configs", "hash3d_small.json")))
B = 32768


def worker(rank, world, out, shard_optimizer, native, peer_memory):
    import oracle_binding as ob
    import tcnn_b200
    from tcnn_b200.dp import DataParallelTrainer

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT="29533")
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    rng = ob.default_rng(1337)
    x = ob.generate_random_uniform(rng, B * 3).reshape(B, 3)
    y = ob.make_targets(x, 3)
    model = tcnn_b200.create_from_config(3, 3, CFG)
    dp = DataParallelTrainer(model.trainer, shard_optimizer=shard_optimizer, native=native, peer_memory=peer_memory)
    assert dp.native == native and dp.shard_optimizer == shard_optimizer
    if rank == 0:
        print("engine:", dp.engine, flush=True)
    if peer_memory and os.environ.get("TCNNB_REQUIRE_PEER_MEMORY"):
        assert dp.engine.startswith("peer-memory"), dp.engine
    lo, hi = dp.shard(B)
    xd, yd = torch.from_numpy(x[lo:hi]).cuda(), torch.from_numpy(y[lo:hi]).cuda()
    losses = []
    for _ in range(5):
        dp.training_step(xd, yd)
        losses.append(dp.loss())
    dp.sync_full_precision()
    torch.cuda.synchronize()
    np.savez(os.path.join(out, f"dp{rank}_{int(shard_optimizer)}{int(native)}{int(peer_memory)}.npz"), p=model.trainer.params_full_precision().cpu().numpy(), p16=model.trainer.params().cpu().view(torch.int16).numpy(), losses=np.array(losses))
    dp.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    import tempfile

    out = tempfile.mkdtemp(prefix="dp_parity_")  # the ranks' parameters and losses, compared below
    # (sharded optimizer, native engine inside libtcnn_b200, peer-memory kernels instead of NCCL collectives)
    MODES = [(False, False, False), (True, False, False), (False, True, False), (True, True, False), (True, True, True)]
    WORLD = int(os.environ.get("TCNNB_DP_WORLD", "2"))
    if os.environ.get("TCNNB_DP_MODES"):  # e.g. "4" = the peer-memory engine only (8-GPU runs are charged 8x)
        MODES = [MODES[int(i)] for i in os.environ["TCNNB_DP_MODES"].split(",")]
    for so, nat, pm in MODES:
        mp.spawn(worker, args=(WORLD, out, so, nat, pm), nprocs=WORLD, join=True)
    import oracle_binding as ob
    import tcnn_b200

    torch.cuda.set_device(0)
    rng = ob.default_rng(1337)
    x = ob.generate_random_uniform(rng, B * 3).reshape(B, 3)
    y = ob.make_targets(x, 3)
    model = tcnn_b200.create_from_config(3, 3, CFG)
    xd, yd = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    losses = []
    for _ in range(5):
        model.trainer.training_step(xd, yd)
        losses.append(model.trainer.loss())
    p1 = model.trainer.params_full_precision().cpu().numpy()
    for so, nat, pm in MODES:
        r0, r1 = np.load(os.path.join(out, f"dp0_{int(so)}{int(nat)}{int(pm)}.npz")), np.load(os.path.join(out, f"dp{WORLD - 1}_{int(so)}{int(nat)}{int(pm)}.npz"))
        print("sharded optimizer:", so, "native engine:", nat, "peer memory:", pm)
        print("  replicas identical (fp32 masters / fp16 working):", np.array_equal(r0["p"], r1["p"]), np.array_equal(r0["p16"], r1["p16"]))
        print("  losses dp:", r0["losses"].tolist())
        print("  losses 1gpu:", losses)
        print("  max |param diff| dp vs 1gpu:", float(np.abs(r0["p"] - p1).max()), "mean:", float(np.abs(r0["p"] - p1).mean()))
        assert np.array_equal(r0["p"], r1["p"]) and np.array_equal(r0["p16"], r1["p16"])
        assert np.allclose(r0["losses"], losses, rtol=2e-2)
    print("DP PARITY OK")
