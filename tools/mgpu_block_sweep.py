"""Multi-GPU tuning aid (torchrun, N GPUs): C3 trust-region iterations with the column-distributed factorisation for several
ownership block sizes (COVINS_B200_DIST_BLOCK = consecutive pose tile columns per owner)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import covins_b200
from covins_b200 import optimization as O, synth_map

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
import datetime
dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=datetime.timedelta(seconds=int(os.environ.get("COVINS_NCCL_TIMEOUT", "90"))))
ctx = covins_b200.Context(local)
cfg = sys.argv[1] if len(sys.argv) > 1 else "C3"
p = synth_map.make_config(cfg)
for spec in (sys.argv[2].split(",") if len(sys.argv) > 2 else "1,2,3,4,6,8".split(",")):
    os.environ["COVINS_B200_DIST_BLOCK"] = str(int(spec))
    s = O.BaSolver(ctx, p, rank=rank, world=world, allreduce=O.torch_allreduce(), p2p=True)
    s.iterate(2); ctx.sync(); dist.barrier()
    s.restart(); s.timing(reset=True); ctx.sync(); dist.barrier()
    t0 = time.perf_counter()
    n = s.iterate(8); ctx.sync()
    dt = time.perf_counter() - t0
    r = s.result(); tm = s.timing(); s.close()
    it = max(r["iterations"], 1)
    if rank == 0:
        print(f"{cfg} world={world} p2p={'on' if s.p2p else 'off'} block={spec}: {1e3 * dt / max(n, 1):.2f} ms/it (factor {tm['factor_ms']/it:.2f}, "
              f"blocks+schur+exchange {tm['build_schur_ms']/it:.2f}, solve {tm['solve_ms']/it:.2f}) final cost {r['final_cost']:.6f}", flush=True)
    dist.barrier()
dist.destroy_process_group()
