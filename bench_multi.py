"""Multi-GPU arm of bench.py (imported when WORLD_SIZE > 1): strong scaling of the SAME frame
(cfg3 by default) over N GPUs of one box, one process per GPU (torchrun), NCCL for the plumbing,
splats exchanged by direct peer-memory stores (web-splat_b200/csrc/shard.cu)."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def run(args):
    import torch
    import torch.distributed as dist
    import bench
    import websplat_b200 as ws
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ.get("LOCAL_RANK", "0"))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device -- the product path has no CPU fallback")
    torch.cuda.set_device(local)
    # NCCL prints its version banner (and any NCCL_DEBUG output) on stdout; the contract is ONE JSON
    # line there, so stdout is parked on stderr until the result is printed
    sys.stdout.flush()
    saved_stdout = os.dup(1)
    os.dup2(2, 1)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    if args.workload == "cfg5":
        # 24 M Gaussians: every rank generates ONLY its own eighth (seeded by rank) -- the union is the cloud; the
        # global bbox / centre the frame needs are reduced over the ranks.  (cfg5 exists only sharded, so there is
        # no single-GPU frame to stay byte-identical with.)
        n_all, W, H, seed, _ = ws.synth.CONFIGS["cfg5"]
        lo_i, hi_i = (n_all * rank) // world, (n_all * (rank + 1)) // world
        shard = ws.synth.make_cloud(hi_i - lo_i, seed + 7919 * rank, density_n=n_all)
        lo = torch.tensor(shard["aabb_min"], device="cuda"); hi = torch.tensor(shard["aabb_max"], device="cuda")
        csum = torch.tensor(shard["center"].astype(np.float64) * (hi_i - lo_i), device="cuda")
        dist.all_reduce(lo, op=dist.ReduceOp.MIN); dist.all_reduce(hi, op=dist.ReduceOp.MAX); dist.all_reduce(csum)
        cloud = dict(shard, num_points=n_all, aabb_min=lo.cpu().numpy(), aabb_max=hi.cpu().numpy(),
                     center=(csum / n_all).cpu().numpy().astype(np.float32))
        shard = dict(shard, aabb_min=cloud["aabb_min"], aabb_max=cloud["aabb_max"], center=cloud["center"])
        views = ws.synth.orbit_views(36)
    else:
        # one process generates the cloud, the others load it (identical bytes on every rank)
        if local == 0:
            cloud, W, H, views = bench.make_workload(args.workload)
        dist.barrier()
        if local != 0:
            cloud, W, H, views = bench.make_workload(args.workload)
        shard = ws.shard_cloud(cloud, rank, world)
    ctx = ws.Context(local)
    gen = ws.GenericGaussianPointCloud(shard["gaussians"], shard["sh_coefs"], shard["sh_deg"], shard["num_points"],
                                       ws.Aabb(cloud["aabb_min"], cloud["aabb_max"]), cloud["center"],
                                       compressed=cloud["compressed"], covars=cloud.get("covars"), quantization=cloud.get("quantization"))
    pc = ws.PointCloud.new(ctx, gen)
    fmt = ws.FORMAT_RGBA16_FLOAT
    N = int(cloud["num_points"])
    depth = int(getattr(args, "frames_in_flight", 0) or 0)
    if depth <= 0:
        # the smaller a GPU's share, the more latency-bound a single frame is and the more frames fit next to each other.
        # The depths come from a sweep of 2-8 frames in flight at cfg3 on 2, 4 and 8 GPUs of the previous target GPU;
        # they have not been re-measured on H100.  A deeper pipeline also ramps up
        # longer, which a short run sees, hence 4 at 8 GPUs.
        depth = 4 if world >= 8 else 3
    pipe = ws.ShardedPipeline(ws, ctx, fmt, cloud["sh_deg"], cloud["compressed"], pc, N, (W, H), depth=depth,
                              pair_capacity=min(max(8 * N // world + (1 << 22), 1 << 22), (1 << 30) - 1))
    sh = pipe.slots[0]                       # slot 0 also serves the single-frame breakdowns below
    fargs = [bench.frame_args(ws, cloud, v, W, H) for v in views]
    K, Wu = args.steps, max(args.warmup, 3)
    host = [torch.empty((H, W, 4), dtype=torch.float16).pin_memory() for _ in range(2)] if rank == 0 else None

    def sync_all():
        torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.synchronize()

    # ---- kernel-only: frame assembled on every rank's device, no host copy ------------------------
    sh.r.set_timing(False)
    # the bands are stored straight into rank 0's assembled frame (peer memory) by the compositor
    for i in range(Wu):
        pipe.frame_peer(fargs[i % len(fargs)])
    sync_all()
    # cost-balanced bands from the pair counts of the warm-up frames (every rank derives the same boundaries)
    bands0 = list(pipe.bands)
    if not getattr(args, "equal_bands", False):
        for _ in range(2):
            pipe.rebalance()
            sync_all()
            # 2 * depth frames: every slot replays BOTH of its frame graphs (one per frame-buffer parity) on the new bands, so
            # that no graph capture / instantiation is left for the timed region
            for i in range(2 * depth):
                pipe.frame_peer(fargs[(Wu + i) % len(fargs)])
            sync_all()
    # ---- parity evidence carried by the line (before anything is timed): the sharded frame of one fixed view, downloaded
    #      on the root, must have the CRC-32 of the SAME view rendered by ONE GPU (rank 0, plain renderer, whole cloud) --
    #      and therefore the value bench.py prints at N = 1
    cview = fargs[bench.CHECKSUM_VIEW % len(fargs)]
    chk = torch.zeros((H, W, 4), dtype=torch.float16).pin_memory() if rank == 0 else None
    pipe.synchronize()
    sync_all()
    sh.frame_peer(cview, host=chk)
    sync_all()
    checksum = checksum_n1 = None
    if rank == 0:
        checksum = bench.frame_crc(chk)
        if args.workload == "cfg5":
            # cfg5 exists only sharded; the union of the ranks' shards IS the cloud (24 M fits one H100): rebuild it here
            parts = [shard if q == 0 else ws.synth.make_cloud((n_all * (q + 1)) // world - (n_all * q) // world, seed + 7919 * q, density_n=n_all)
                     for q in range(world)]
            full = dict(cloud, gaussians=np.concatenate([p_["gaussians"] for p_ in parts]),
                        sh_coefs=np.concatenate([p_["sh_coefs"] for p_ in parts]), num_points=n_all)
            del parts
        else:
            full = cloud
        fgen = ws.GenericGaussianPointCloud(full["gaussians"], full["sh_coefs"], full["sh_deg"], full["num_points"],
                                            ws.Aabb(cloud["aabb_min"], cloud["aabb_max"]), cloud["center"], compressed=cloud["compressed"],
                                            covars=cloud.get("covars"), quantization=cloud.get("quantization"))
        fpc = ws.PointCloud.new(ctx, fgen)
        plain = ws.GaussianRenderer.new(ctx, fmt, cloud["sh_deg"], cloud["compressed"])
        plain.set_pair_capacity(min(max(8 * N, 1 << 22), (1 << 30) - 1))
        plain.set_timing(False)
        plain.prepare(None, fpc, cview)
        plain.render_to_host(chk, fpc)
        torch.cuda.synchronize()
        checksum_n1 = bench.frame_crc(chk)
        del plain, fpc, fgen, full
    sampler = bench.ClockSampler(local) if rank == 0 else None      # NVML init + thread start BEFORE the barrier: rank 0 alone pays
    if sampler:                                                     # them, and the other ranks would wait for it inside their timed region
        sampler.start()
    sync_all()
    if sampler:
        sampler.reset()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    cur = torch.cuda.current_stream()
    e0.record(cur)
    for st in pipe.streams:
        st.wait_event(e0)
    for i in range(K):
        pipe.frame_peer(fargs[(Wu + i) % len(fargs)])
    for st in pipe.streams:
        cur.wait_stream(st)
    e1.record(cur)
    sync_all()
    ms = torch.tensor([e0.elapsed_time(e1)], device="cuda")
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms_total = float(ms.item())
    clocks = sampler.finish() if sampler else None

    # ---- e2e: rank 0 additionally downloads every frame into pinned host memory -------------------
    copy_stream = torch.cuda.Stream() if rank == 0 else None     # root: download frame f while frame f+1 is produced
    host = [torch.empty((H, W, 4), dtype=torch.float16).pin_memory() for _ in range(2 * depth)] if rank == 0 else None
    pipe._i = 0                               # frame i -> slot i % depth, host buffer i % (2 * depth)
    for i in range(2 * depth * ((Wu + 2 * depth - 1) // (2 * depth))):
        pipe.frame_peer(fargs[i % len(fargs)], host=host[i % (2 * depth)] if rank == 0 else None, copy_stream=copy_stream)
    sync_all()
    t0 = time.perf_counter()
    for i in range(K):
        pipe.frame_peer(fargs[(Wu + i) % len(fargs)], host=host[i % (2 * depth)] if rank == 0 else None, copy_stream=copy_stream)
    sync_all()
    e2e = torch.tensor([time.perf_counter() - t0], device="cuda", dtype=torch.float64)
    dist.all_reduce(e2e, op=dist.ReduceOp.MAX)
    e2e_s = float(e2e.item())

    # ---- per-stage breakdown (max over ranks of each stage) ----------------------------------------
    sh.r.set_timing(True)
    keys = ("ms_preprocess", "ms_sort", "ms_blend", "ms_depth_sort", "ms_binning", "ms_tile_sort")
    acc = np.zeros(len(keys)); vv = []; pp = []
    for i in range(min(K, 36)):
        sh.frame_peer(fargs[(Wu + i) % len(fargs)])
        torch.cuda.synchronize()
        s = sh.stats()
        acc += [s[k] for k in keys]; vv.append(s["num_visible"]); pp.append(s["num_pairs"])
    acc /= min(K, 36)
    t = torch.tensor(list(acc) + [float(np.mean(vv)), float(np.mean(pp))], device="cuda", dtype=torch.float64)
    tmax = t.clone(); dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
    tsum = t.clone(); dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
    # ---- phase timeline of the sharded frame (events between the phases, rank 0's view) ------------
    phases = {}
    for i in range(12):
        marks = []
        dist.barrier()
        sh.frame_to_root(fargs[(Wu + i) % len(fargs)], marks=marks)
        torch.cuda.synchronize()
        for (la, ea), (lb, eb) in zip(marks[:-1], marks[1:]):
            phases[lb] = phases.get(lb, 0.0) + ea.elapsed_time(eb) / 12.0
    if rank == 0:
        peak, peak_src, _ = bench.measured_peaks()
        fps = K / (ms_total * 1e-3)
        stage = {k[3:]: float(tmax[i]) for i, k in enumerate(keys)}
        V_sum, P_sum = float(tsum[-2]), float(tsum[-1])
        T = ((W + 15) // 16) * ((H + 15) // 16)
        bytes_sort_blend = 4 * V_sum * 16 + V_sum * 12 + P_sum * 8 + 2 * P_sum * 16 + P_sum * 24 + W * H * 8
        sb_ms = stage["sort"] + stage["blend"]
        line = {
            "metric": bench.METRIC, "value": fps, "unit": "frames/s", "n_gpus": world, "steps": K, "warmup": Wu,
            "ms_per_step": ms_total / K, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": bench.workload_name(args.workload, cloud, W, H), "target_format": "rgba16float",
                       "parallelism": "stage 1 sharded by Gaussian index, stages 2-3 by tile-row band; splats, count rows, barriers and the finished bands all move by peer-memory stores (no NCCL call inside a frame)",
                       "frames_in_flight": depth, "bands_tile_rows": list(pipe.bands), "bands_equal_split": bands0,
                       "l2": "inputs larger than L2; no flush needed", "N": N, "V_received_sum": V_sum, "P_sum": P_sum, "tiles": T},
            "ms_per_frame": {"preprocess+exchange": stage["preprocess"], "sort": stage["sort"], "blend": stage["blend"],
                             "depth_sort": stage["depth_sort"], "binning": stage["binning"], "tile_sort": stage["tile_sort"],
                             "note": "max over ranks of each stage", "phases_rank0": phases},
            "roofline": {"kernel": "sort+blend (all ranks)", "bound": "hbm", "achieved": bytes_sort_blend / (sb_ms * 1e-3) / 1e9 if sb_ms > 0 else 0.0,
                         "peak": peak * world, "unit": "GB/s", "frac": (bytes_sort_blend / (sb_ms * 1e-3) / 1e9) / (peak * world) if sb_ms > 0 else 0.0,
                         "peak_source": peak_src + " x n_gpus"},
            "cpu_baseline": None,
            "e2e": {"value": K / e2e_s, "unit": "frames/s", "h2d_bytes_per_step": 480 * world, "d2h_bytes_per_step": W * H * 8,
                    "checksum": checksum, "checksum_what": "CRC-32 of the full RGBA16F frame of view %d, assembled from the %d ranks' bands and downloaded on rank 0" % (bench.CHECKSUM_VIEW, world),
                    "checksum_n1_same_view": checksum_n1, "checksum_matches_n1": checksum == checksum_n1},
            # per rank and frame: epoch 1 + stage 1 3 + routing 3 (+ 2 gate kernels with several frames in flight) + finish / histogram 1 +
            # depth passes 4 + per depth slab (binning 3 + tile passes 2 + composite 1); + the root's wait for the bands
            "gpu_launches": K * (world * (12 + (2 if depth > 1 else 0) + (2 if (N // world) >= 2_000_000 else 1) * 6) + 1),
            "clocks": clocks,
        }
        sys.stdout.flush()
        os.dup2(saved_stdout, 1)
        print(json.dumps(line), flush=True)
        os.dup2(2, 1)
    dist.barrier()
    dist.destroy_process_group()
    return 0
