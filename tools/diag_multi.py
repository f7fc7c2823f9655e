"""N-rank diagnosis of the sharded forward (run with torchrun on an N-GPU node):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29544 tools/diag_multi.py

Every rank renders (1) the whole image and (2) its slab on ITS OWN GPU and compares them locally (is a rank's slab render
different from its whole render?); rank 0 then compares its whole image with every other rank's whole image (do the GPUs /
processes agree?), and the all-reduced slab sum with its whole image (is the collective exact?).  Open issue of round 1:
at 8 ranks the gathered colour map differed from the single-GPU one by 1.5e-3 in a few pixels while 8 slabs on one GPU
compose bit-exactly (tools/diag_slabs.py)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "rade-gs_b200"))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import diff_gaussian_rasterization as dgr  # noqa: E402
from rade_gs_b200 import multigpu, scenes  # noqa: E402

rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
local = int(os.environ.get("LOCAL_RANK", rank))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
if world > 1:
    dist.init_process_group("nccl", device_id=dev)
C = dgr._C
sc = scenes.make_scene(60000, 640, 400, 500.0, -3.8, seed=21, view=scenes.look_at_view((0.3, 0.2, -0.4), (0.0, 0.1, 6.0)), bg=(0.2, 0.1, 0.3)).to(dev)
E = torch.Tensor([])
args = (sc.bg, sc.means3D, E, sc.opacities, sc.scales, sc.rotations, 1.0, E, sc.viewmatrix, sc.projmatrix, sc.tanfovx, sc.tanfovy, 0.1, sc.height,
        sc.width, sc.shs, 3, sc.campos, False, True, True, False)
gy = (sc.height + 15) // 16
b, e = multigpu.partition_tile_rows(gy, world)[rank]
slab = C.rasterize_gaussians_slab(*args, b, e)     # slab first: nothing from a whole-image call can be lying around in memory
whole = C.rasterize_gaussians(*args)
names = {1: "color", 2: "coord", 4: "alpha", 5: "normal", 6: "depth"}
local_bad = {n: int((slab[i][:, b * 16: e * 16] != whole[i][:, b * 16: e * 16]).sum()) for i, n in names.items()}
outside = {n: int((slab[i][:, : b * 16] != 0).sum() + (slab[i][:, e * 16:] != 0).sum()) for i, n in names.items()}
print(f"[rank {rank}] slab {b}-{e}: slab-vs-own-whole mismatches {local_bad}, nonzero outside slab {outside}", flush=True)
if world > 1:
    for i, n in names.items():
        mine = whole[i].clone()
        ref = whole[i].clone()
        dist.broadcast(ref, src=0)
        cross = int((mine != ref).sum())
        summed = slab[i].clone()
        dist.all_reduce(summed)
        coll = int((summed != whole[i]).sum())
        gathered = [torch.empty_like(slab[i]) for _ in range(world)]
        dist.all_gather(gathered, slab[i])
        manual = torch.stack(gathered).sum(0)
        man = int((manual != whole[i]).sum())
        print(f"[rank {rank}] {n}: whole differs from rank 0's in {cross} elements; all_reduce(slabs) vs own whole: {coll}; all_gather+sum vs own whole: {man}",
              flush=True)
        if (coll or man or cross) and rank == 0:
            bad = torch.nonzero((summed != whole[i]) | (manual != whole[i]) | (mine != ref))[:6]
            for c, y, x in bad.tolist():
                print(f"    {n}[{c},{y},{x}] (tile row {y // 16}): whole {whole[i][c, y, x].item():.9g} all_reduce {summed[c, y, x].item():.9g} gather-sum {manual[c, y, x].item():.9g}"
                      f" per-rank slab values {[round(t[c, y, x].item(), 9) for t in gathered]}", flush=True)
    dist.destroy_process_group()
