"""Timings of the Z-sharded labelling (dist.label) and of dist.fill_holes_auto, one JSON line on rank 0.

    python -m torch.distributed.run --nproc-per-node N tools/bench_dist_label.py [--sizes 512,1024] [--c5]

One rank per GPU over NCCL when the box has N GPUs; with fewer GPUs the ranks share them over gloo
(tensors staged through the host), which the JSON reports. Workloads: the bone mask (226..3071) of
phantom.ct at each size, and its complement (one giant component), 26-connected; fill_holes_auto runs
on the bone mask at conn 6, size 1000. Per stage, the median over --reps of the slowest rank, from CUDA
events around the backend calls: local labelling (b2v_label on the slab), boundary forest, resolve
(union-find + lookup table), relabel; "exchange" is the rest of dist.label (the four collectives and
their host work; for fill_holes_auto also the mask reset, the histogram, its all_reduce and the
apply). Every result is verified against labeling.label_device / labeling.fill_holes_auto on
the gathered volume on rank 0. --c5 adds the 1024 x 2048 x 2048 volume (2^32 voxels, beyond the
single-GPU labelling; needs 3 ranks or more), checked by invariants instead: the labels cover exactly
the foreground, every label in 1..total is used, and foreground neighbours across every boundary carry
equal labels. The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
from bench_mask_editor import card  # noqa: E402
from scipy.ndimage import generate_binary_structure  # noqa: E402
from invesalius3_b200 import device as dev, dist as zd, labeling, phantom  # noqa: E402

STAGES = ("local", "boundary", "resolve", "relabel")


class TimedBackend(zd.DeviceBackend):
    """DeviceBackend with CUDA events around each labelling stage."""

    def __init__(self):
        super().__init__()
        self.ev = {}

    def _timed(self, stage, fn, *a):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); out = fn(*a); e1.record()
        self.ev[stage] = (e0, e1)
        return out

    def lb_local(self, *a):
        return self._timed("local", super().lb_local, *a)

    def lb_boundary(self, *a):
        return self._timed("boundary", super().lb_boundary, *a)

    def lb_resolve(self, *a):
        return self._timed("resolve", super().lb_resolve, *a)

    def lb_relabel(self, *a):
        return self._timed("relabel", super().lb_relabel, *a)

    def times(self):
        torch.cuda.synchronize()
        t = {s: (self.ev[s][0].elapsed_time(self.ev[s][1]) if s in self.ev else 0.0) for s in STAGES}
        self.ev = {}
        return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="512,1024")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--c5", action="store_true")
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    ngpu = torch.cuda.device_count()
    torch.cuda.set_device(local % ngpu)
    backend = "nccl" if ngpu >= int(os.environ.get("LOCAL_WORLD_SIZE", world)) else "gloo"
    if backend == "nccl":       # one rank too: dist.label gathers through the process group
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    else:
        dist.init_process_group("gloo")
    real_stdout = os.fdopen(os.dup(1), "w"); os.dup2(2, 1)
    be = TimedBackend()
    s26 = generate_binary_structure(3, 3)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()

    def slowest(x):
        t = torch.tensor([x], dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def run(fn):
        """Median over reps of the slowest rank: total and per-stage ms."""
        fn()
        be.times()
        rows = []
        for _ in range(args.reps):
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); out = fn(); e1.record()
            torch.cuda.synchronize()
            st = be.times()
            total = e0.elapsed_time(e1)
            row = {"total_ms": slowest(total)}
            for s in STAGES:
                row[f"{s}_ms"] = slowest(st[s])
            row["exchange_ms"] = slowest(total - sum(st.values()))
            rows.append(row)
        return {k: round(float(np.median([r[k] for r in rows])), 3) for k in rows[0]}, out

    def gather(own, DZ):
        """The whole volume on rank 0 (None elsewhere)."""
        if world == 1:
            return own
        shard = zd.ZShard(DZ, rank, world)
        if rank == 0:
            whole = torch.empty((DZ,) + tuple(own.shape[1:]), dtype=own.dtype, device="cuda")
            whole[: own.shape[0]].copy_(own)
            for r in range(1, world):
                a, b = shard.bounds(r)
                if backend == "nccl":
                    dist.recv(whole[a:b].view(torch.uint8), src=r)
                else:
                    buf = torch.empty(whole[a:b].view(torch.uint8).shape, dtype=torch.uint8)
                    dist.recv(buf, src=r)
                    whole[a:b].view(torch.uint8).copy_(buf)
            return whole
        dist.send(own.contiguous().view(torch.uint8) if backend == "nccl" else own.cpu().contiguous().view(torch.uint8),
                  dst=0)
        return None

    results = []
    for n in (int(s) for s in args.sizes.split(",") if s):
        shard = zd.ZShard(n, rank, world)
        img = torch.from_numpy(phantom.ct((n, n, n), seed=2, zrange=(shard.z0, shard.z1))).cuda()
        bone = dev.threshold(img, 226, 3071)
        del img
        for name, fg in ((f"bone_{n}", bone), (f"bone_{n}_complement", (bone == 0).to(torch.uint8))):
            tm, (lab, total) = run(lambda: zd.label(fg, s26, shard, backend=be))
            res = {"input": name, "shape": [n, n, n], "labels": total, **tm}
            whole_fg, whole_lab = gather(fg, n), gather(lab, n)
            if rank == 0:
                want, wn = labeling.label_device(whole_fg, s26)
                res["verified"] = bool(wn == total and torch.equal(want, whole_lab))
                del want
            del whole_fg, whole_lab, lab
            results.append(res)
        src = bone.clone()
        m = bone.clone()

        def fill():
            m.copy_(src)
            return zd.fill_holes_auto(m, 6, 1000, shard, backend=be)
        tm, ret = run(fill)
        res = {"input": f"fill_holes_auto_bone_{n}", "shape": [n, n, n], "conn": 6, "size": 1000, "filled": ret, **tm}
        whole_src, whole_m = gather(src, n), gather(m, n)
        if rank == 0:
            want = whole_src.cpu().numpy()
            wret = labeling.fill_holes_auto(want, 6, 1000)
            res["verified"] = bool(wret == ret and np.array_equal(want, whole_m.cpu().numpy()))
        del whole_src, whole_m, src, m, bone
        torch.cuda.empty_cache()
        results.append(res)

    if args.c5 and world >= 3:
        from configs_multigpu import phantom_planes
        DZ, dy, dx = 1024, 2048, 2048
        shard = zd.ZShard(DZ, rank, world)
        bone = dev.threshold(phantom_planes(DZ, dy, dx, shard.z0, shard.z1, 5), 226, 3071)
        for name, fg in (("c5_bone", bone), ("c5_bone_complement", (bone == 0).to(torch.uint8))):
            tm, (lab, total) = run(lambda: zd.label(fg, s26, shard, backend=be))
            res = {"input": name, "shape": [DZ, dy, dx], "labels": total, **tm}
            lab_u = lab.view(torch.int32)
            ok = bool(torch.equal(lab_u != 0, fg != 0))
            used = torch.zeros(total + 1, dtype=torch.int32, device="cuda")
            used.index_fill_(0, lab_u.reshape(-1).to(torch.int64), 1)
            counts = torch.tensor([int((lab_u != 0).sum()), int((fg != 0).sum())], dtype=torch.int64, device="cuda")
            if world > 1:
                for t, op in ((used, dist.ReduceOp.MAX), (counts, dist.ReduceOp.SUM)):
                    h = t if backend == "nccl" else t.cpu()
                    dist.all_reduce(h, op=op)
                    t.copy_(h)
            ok = ok and bool(used[1:].all()) and int(counts[0]) == int(counts[1])
            # foreground neighbours across the boundary below this shard's last plane carry equal labels
            first = lab[0].contiguous()
            hi = torch.empty_like(first)
            ops = []
            if shard.has_lo:
                ops.append(dist.P2POp(dist.isend, first if backend == "nccl" else first.cpu(), rank - 1))
            if shard.has_hi:
                hi = hi if backend == "nccl" else hi.cpu()
                ops.append(dist.P2POp(dist.irecv, hi, rank + 1))
            if ops:
                for q in dist.batch_isend_irecv(ops):
                    q.wait()
            if shard.has_hi:
                lo, hi = lab[-1], hi.cuda()
                for oy in (-1, 0, 1):
                    for ox in (-1, 0, 1):
                        a = lo[max(0, -oy): dy - max(0, oy), max(0, -ox): dx - max(0, ox)]
                        b = hi[max(0, oy): dy + min(0, oy), max(0, ox): dx + min(0, ox)]
                        both = (a != 0) & (b != 0)
                        ok = ok and bool(torch.equal(a[both], b[both]))
            res["verified"] = slowest(0.0 if ok else 1.0) == 0.0
            del lab, used
            results.append(res)
        del bone
    if rank == 0:
        name, plim = card()
        out = {"metric": "dist_label", "gpu": name, "power_limit": plim, "ranks": world, "gpus": ngpu,
               "collectives": backend, "reps": args.reps, "results": results,
               "verified": all(r["verified"] for r in results)}
        real_stdout.write(json.dumps(out) + "\n")
        real_stdout.flush()
    dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
