#!/usr/bin/env python
"""bench.py - LiDAR frames/sec of the SST hot path (BASELINE.json metric) on N H100s of one node.

A "step" = one forward of BASELINE config 2 per GPU: 1 synthetic Waymo-shaped sweep (150k pts, 0.32 m pillars,
~30k non-empty) through dynamic voxelisation -> DynamicVFE -> SSTInputLayerV2 -> SSTv2 (6 blocks = 12 SRA
layers, d=128, h=8, ff=256), sparse output (to_bev=False, no attached convs).  Frames shard over GPUs
(weak scaling, no data-path collective: inference has none, SURVEY.md 8e).

    python bench.py --gpus 1 --steps 20 --warmup 5
    python bench.py --gpus 1 --steps 20 --warmup 5 --dump-outputs DIR   # + the last timed step's outputs as DIR/*.npy
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...
    python bench.py --impl reference          # CPU port of the reference path on the host cores
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

P_POINTS = 150000
METRIC = "lidar_frames_per_sec_sst6_fwd_150k"
# one workload string for both arms (the driver compares them)
WORKLOAD = "config2: SST-6 fwd, 150k-pt Waymo-shaped sweep, 0.32m pillars, d=128 h=8 ff=256, batch 1 per GPU, sparse output"


def peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm=d["hbm_gbs"], tf_burst=d["bf16_tflops"], tf_sustained=d["bf16_tflops_sustained"], src="measured")
    # NVIDIA H100 SXM data sheet (700 W card; a card set to a lower power limit sustains less): 3.35 TB/s, 989 TFLOP/s dense fp16/bf16
    return dict(hbm=3350.0, tf_burst=989.0, tf_sustained=989.0, src="H100 SXM data sheet")


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        self.idx, self.rows, self.proc, self.windows = gpu_index, [], None, []

    def begin(self):
        """Open a timed window: only samples that arrive inside a window count (the sampler itself is started earlier,
        because nvidia-smi needs tens of ms to produce its first line)."""
        self.windows.append([time.time(), None])

    def end(self):
        self.windows[-1][1] = time.time()

    def start(self):
        """NVML in-process (ready when start() returns; a fresh box can take > 1 s to bring up an `nvidia-smi -lms` child, longer than
        the whole timed region); the nvidia-smi loop stays as the fallback."""
        self.mode, self.proc, self.running = None, None, False
        try:
            import pynvml as N
            N.nvmlInit()
            try:
                uuid = str(torch.cuda.get_device_properties(self.idx).uuid)
                self.h = N.nvmlDeviceGetHandleByUUID(uuid if uuid.startswith("GPU-") else "GPU-" + uuid)
            except Exception:
                self.h = N.nvmlDeviceGetHandleByIndex(self.idx)
            N.nvmlDeviceGetClockInfo(self.h, N.NVML_CLOCK_SM)
            self.N, self.mode, self.running = N, "nvml", True
            self.t = threading.Thread(target=self._poll, daemon=True)
            self.t.start()
            return
        except Exception:
            pass
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                          "-i", str(self.idx), "-lms", "10"], stdout=subprocess.PIPE,
                                         stderr=subprocess.DEVNULL, text=True)
            self.mode = "nvidia-smi"
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _poll(self):
        N = self.N
        bits = {"hw_slowdown": 0x8, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20, "sw_power_cap": 0x4}   # nvmlClocksEventReason*
        get_reasons = getattr(N, "nvmlDeviceGetCurrentClocksEventReasons", None) or N.nvmlDeviceGetCurrentClocksThrottleReasons
        while self.running:
            try:
                sm, mx = N.nvmlDeviceGetClockInfo(self.h, N.NVML_CLOCK_SM), N.nvmlDeviceGetMaxClockInfo(self.h, N.NVML_CLOCK_SM)
                r = int(get_reasons(self.h))
                row = ["", str(sm), str(mx), "", ""] + ["Active" if r & bits[k] else "Not Active"
                                                        for k in ("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap")]
                self.rows.append((time.time(), row))
            except Exception:
                pass
            time.sleep(0.004)

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append((time.time(), [x.strip() for x in line.split(",")]))

    def stop(self):
        if self.mode is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no clock source (pynvml / nvidia-smi unavailable)"], "samples": 0}
        self.running = False
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                self.proc.kill()

        def collect(inside_only):
            sm, mx, reasons = [], [], set()
            for ts, r in self.rows:
                if inside_only and self.windows and not any(a <= ts <= (b if b is not None else ts) for a, b in self.windows):
                    continue
                try:
                    sm.append(float(r[1]))
                    mx.append(float(r[2]))
                    for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[5:9]):
                        if v.lower().startswith("active"):
                            reasons.add(name)
                except Exception:
                    pass
            return sm, mx, reasons
        sm, mx, reasons = collect(True)
        where = "inside the timed windows"
        if not sm:   # the source delivered nothing while the windows were open: report what it saw around them, and say so
            sm, mx, reasons = collect(False)
            where = "around the timed windows (none fell inside)"
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm), "source": f"{self.mode}, samples {where}"}


_BEST_THREADS = None


def pick_threads():
    """Intra-op thread count that makes the CPU path fastest on this host (many small ops: all cores is not
    always best).  Tried: 8, 16, 32, all; measured on a 20k-point frame; cached."""
    global _BEST_THREADS
    if _BEST_THREADS is not None:
        return _BEST_THREADS
    from oracle import sst_oracle as O
    from sst_b200 import flagship as fl
    ncpu = os.cpu_count() or 1
    cands = sorted({min(ncpu, t) for t in (8, 16, 32, ncpu)})
    cfg = fl.sst_cfg(num_blocks=2)
    vfe, il, bb = fl.build_sst(cfg)
    wv, wb = dict(vfe.state_dict()), dict(bb.state_dict())
    pts = O.synth_frame(1, 40000)
    best = (1e30, ncpu)
    with torch.no_grad():
        for t in cands:
            torch.set_num_threads(t)
            for rep in range(2):
                t0 = time.perf_counter()
                co = torch.nn.functional.pad(O.dynamic_voxelize(pts, fl.VOXEL_SIZE, fl.PC_RANGE), (1, 0), value=0)
                vf, vc = O.dynamic_vfe_forward(pts, co, wv, fl.VOXEL_SIZE, fl.PC_RANGE, 2)
                info = O.input_layer_v2(vf, vc, fl.DROP_TEST, fl.WINDOW_SHAPE, (468, 468, 1))
                O.sstv2_forward(info, wb, cfg['backbone']['nhead'], 2)
                dt = time.perf_counter() - t0
            best = min(best, (dt, t))
    _BEST_THREADS = best[1]
    return _BEST_THREADS


def cpu_oracle_frames(n_frames, warmup, threads=None, budget_s=None):
    """The reference's own CPU path (restated in oracle/, see oracle/sst_oracle.py header) on the host cores.  `budget_s`
    bounds the sample: no new frame is started once the timed frames have used that many seconds."""
    from oracle import sst_oracle as O
    from sst_b200 import flagship as fl
    threads = threads or pick_threads()
    torch.set_num_threads(threads)
    cfg = fl.sst_cfg()
    vfe, il, bb = fl.build_sst(cfg)
    wv, wb = dict(vfe.state_dict()), dict(bb.state_dict())
    times = []
    with torch.no_grad():
        for i in range(warmup + n_frames):
            pts = O.synth_frame(1000 + i, P_POINTS)
            t0 = time.perf_counter()
            co = torch.nn.functional.pad(O.dynamic_voxelize(pts, fl.VOXEL_SIZE, fl.PC_RANGE), (1, 0), value=0)
            vf, vc = O.dynamic_vfe_forward(pts, co, wv, fl.VOXEL_SIZE, fl.PC_RANGE, 2)
            info = O.input_layer_v2(vf, vc, fl.DROP_TEST, fl.WINDOW_SHAPE, (468, 468, 1))
            out = O.sstv2_forward(info, wb, cfg['backbone']['nhead'], cfg['backbone']['num_blocks'])
            dt = time.perf_counter() - t0
            if i >= warmup:
                times.append(dt)
                if budget_s is not None and sum(times) >= budget_s:
                    break
    return times, threads, out.shape[0]


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    steps = max(1, args.steps)
    warmup = max(args.warmup, 3)
    # every step is one full frame (~1.5 s on this class of host): K + W frames fit the few-minute budget for the default K = 20;
    # a safety budget still bounds absurd K (the line then says how many frames were timed)
    times, threads, M = cpu_oracle_frames(steps, warmup, budget_s=float(os.environ.get("SSTB200_REF_BUDGET_S", "150")))
    tot = sum(times)
    timed = len(times)
    v = timed / tot
    line = {
        "impl": "reference", "metric": METRIC, "value": v, "unit": "frames/s", "n_gpus": args.gpus, "steps": steps,
        "warmup": warmup, "ms_per_step": 1e3 * tot / timed, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD},
        "cpu_baseline": {"value": v, "unit": "frames/s", "cores": threads, "kind": "port",
                         "sample": f"{timed} of {steps} frames timed after {warmup} warm-up frames (each step = one full config-2 forward) on {threads} host threads, torch CPU fp32; "
                                   "the reference itself is Python and cannot travel to the GPU box, so its restatement oracle/sst_oracle.py (validated bit-exact against it) is timed"},
        "e2e": {"value": v, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line))


def train_bench(args, world, rank, dev, frames_d):
    """BASELINE config 4 on this node: `--train-frames` config-2 sweeps per GPU and step (4 per GPU = 32 frames on 8 GPUs),
    training-mode modules (train drop_info, voxel shuffle, batch-statistics naiveSyncBN with its all-reduce, bf16 GEMM operands),
    loss = mean(out^2), backward through the library's own kernels, ONE NCCL all-reduce over the flat gradient buffer, fused AdamW.
    Timed with CUDA events over the whole step, MAX over ranks; the all-reduce is timed by its own event pair."""
    import torch.distributed as dist
    from sst_b200 import flagship as fl
    from sst_b200.train import TrainStep
    cfg = fl.sst_cfg()
    cfg["backbone"]["precision"] = "bf16"
    cfg["middle_encoder"]["shuffle_voxels"] = True
    vfe, il, bb = fl.build_sst(cfg, seed=0)        # same init on every rank (DDP broadcasts rank 0's weights)
    ts = TrainStep(vfe.to(dev), il, bb.to(dev), fl.VOXEL_SIZE, fl.PC_RANGE)
    B = max(1, args.train_frames)
    K, W = max(2, min(args.steps, 6)), 2
    batches = [[frames_d[(i * B + j) % len(frames_d)] for j in range(B)] for i in range(K + W)]
    for i in range(W):
        ts.step(batches[i])
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    ts.ar_events.clear()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    loss = None
    for i in range(K):
        loss = ts.step(batches[W + i], time_allreduce=True)
    e1.record()
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    ms = e0.elapsed_time(e1)
    ar_ms = sum(a.elapsed_time(b) for a, b in ts.ar_events)
    t = torch.tensor([ms, ar_ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms, ar_ms = float(t[0]), float(t[1])
    nbytes = ts.grad_bytes
    return {"metric": "lidar_frames_per_sec_sst6_train_150k", "value": world * B * K / (ms / 1e3), "unit": "frames/s",
            "frames_per_gpu_per_step": B, "steps": K, "warmup": W, "ms_per_step": ms / K, "dtype": "bf16 operands, fp32 accumulate / master weights",
            "allreduce_ms_per_step": ar_ms / K, "allreduce_share": ar_ms / ms if ms > 0 else None,
            "nccl_gradient_bytes_per_step": nbytes, "nccl_wire_bytes_per_rank_per_step": int(2 * (world - 1) / world * nbytes),
            "collectives_per_step": "1 flat gradient all-reduce + 2 naiveSyncBN statistic all-reduces (fwd) + 2 (bwd)" if world > 1 else "none (1 GPU)",
            "loss": float(loss), "optimizer": "AdamW (fused kernel over one flat buffer)", "scaling": "weak"}


def dump_outputs(out_dir, result):
    """The arrays a caller of SSTEngine.run() receives from the last timed step: the voxel count, the [M, d] voxel features and
    the [M, 4] (batch, z, y, x) coordinates of its M voxels (float64 / float32; < 64 MB for a 150k-point sweep)."""
    import numpy as np
    feats, coors, num = result
    torch.cuda.synchronize()
    M = int(num.item())
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "num_voxels.npy"), np.array([M], dtype=np.float64))
    np.save(os.path.join(out_dir, "voxel_feats.npy"), feats[:M].float().cpu().numpy())
    np.save(os.path.join(out_dir, "voxel_coors.npy"), coors[:M].cpu().numpy().astype(np.float64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--precision", default=os.environ.get("SSTB200_PRECISION", "auto"))
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-fp32", action="store_true", help="skip the fp32-tolerance sub-record")
    ap.add_argument("--no-train", action="store_true", help="skip the training-step sub-record (BASELINE config 4)")
    ap.add_argument("--no-fsd", action="store_true", help="skip the FSD sparse U-Net sub-record (SURVEY 8f next-1)")
    ap.add_argument("--train-frames", type=int, default=4, help="frames per GPU and training step (config 4: 32 frames / 8 GPUs)")
    ap.add_argument("--streams", type=int, default=int(os.environ.get("SSTB200_STREAMS", "8")),
                    help="frames in flight per GPU (independent engines on their own CUDA streams); 1 = strictly serial")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what the last timed step returned (voxel features, coordinates, count) as DIR/<name>.npy")
    args = ap.parse_args()
    if args.impl == "reference":
        return run_reference(args)
    args.warmup = max(args.warmup, 3)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    import torch.distributed as dist
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device(f"cuda:{local}"))
    dev = torch.device(f"cuda:{local}")
    torch.cuda.set_device(dev)
    from sst_b200.dist_utils import pin_to_gpu_numa
    all_cpus = os.sched_getaffinity(0)
    numa_cpus = pin_to_gpu_numa(local)   # host thread + pinned staging buffers on the GPU's NUMA node (None: topology not exposed)

    from sst_b200 import build, flagship as fl
    build.build()
    from sst_b200.engine import SSTEngine

    cfg = fl.sst_cfg()
    vfe, il, bb = fl.build_sst(cfg)
    precision = args.precision
    if precision == "auto":
        precision = "bf16"
    S = max(1, args.streams)
    vfe, bb = vfe.to(dev), bb.to(dev)
    engs = [SSTEngine(fl.VOXEL_SIZE, fl.PC_RANGE, vfe, il, bb, max_points=P_POINTS, batch_size=1, precision=precision, device=dev)
            for _ in range(S)]
    eng = engs[0]

    # inputs larger than L2: NF distinct resident sweeps (1.8 MB each, > 126 MB in total) are cycled, so no timed step
    # finds its input in L2; weights (3 MB) are legitimately L2-resident in steady state.
    NF = 80
    base_frames = [fl.synth_frame(1000 + rank * 8 + i, P_POINTS) for i in range(8)]
    frames_h = base_frames
    g = torch.Generator().manual_seed(7 + rank)
    frames_d = []
    for i in range(NF):   # distinct data per slot: a seeded rigid rotation of one of 8 generated sweeps (cheap, still LiDAR-like)
        f = base_frames[i % 8].clone()
        th = float(torch.rand(1, generator=g)) * 6.283185307179586
        c_, s_ = torch.cos(torch.tensor(th)), torch.sin(torch.tensor(th))
        x, y = f[:, 0].clone(), f[:, 1].clone()
        f[:, 0], f[:, 1] = c_ * x - s_ * y, s_ * x + c_ * y
        frames_d.append(f.to(dev))
    offs_d = torch.tensor([0, P_POINTS], dtype=torch.int32, device=dev)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def step(i):
        e = engs[i % S]
        e.load_frames_device(frames_d[i % NF], offs_d)
        return e.run()

    sampler = ClockSampler(local)
    sampler.start()   # before the warm-up; samples are kept only inside the timed windows (begin/end)
    for i in range(max(args.warmup, S)):
        step(i)
    barrier()
    sampler.begin()
    main = torch.cuda.current_stream(dev)
    windows = []   # one timed window of exactly --steps steps
    last = None
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(main)
    for e in engs:
        e.stream.wait_event(e0)
    for i in range(args.steps):
        last = step(i)
    for e in engs:
        main.wait_stream(e.stream)
    e1.record(main)
    windows.append((e0, e1))
    barrier()
    sampler.end()
    if args.dump_outputs and rank == 0:
        if last is None:
            raise SystemExit("--dump-outputs needs at least one timed step (--steps >= 1)")
        dump_outputs(args.dump_outputs, last)
    wms = torch.tensor([a.elapsed_time(b) for a, b in windows], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(wms, op=dist.ReduceOp.MAX)   # per window: the slowest rank
    wms = sorted(wms.tolist())
    total_ms = wms[len(wms) // 2]
    value = world * args.steps / (total_ms / 1e3)

    # serial single-stream latency per frame (CUDA events around each step, L2 flushed in between) - reported beside it
    flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
    st = eng.stream
    lat = []
    for i in range(6):
        with torch.cuda.stream(st):
            flush.zero_()
            a, b2 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
        eng.load_frames_device(frames_d[i % NF], offs_d)
        eng.run()
        with torch.cuda.stream(st):
            b2.record(st)
        lat.append((a, b2))
    torch.cuda.synchronize()
    lat_ms = sorted(x.elapsed_time(y) for x, y in lat[1:])
    latency_ms = lat_ms[len(lat_ms) // 2]

    # ---- e2e through the public engine API with HOST buffers (H2D + D2H inside the timed region) -------------
    pin = [f.pin_memory() for f in frames_h]
    offs_pin = torch.tensor([0, P_POINTS], dtype=torch.int32).pin_memory()
    outs = [(torch.empty((P_POINTS, eng.d), dtype=torch.float32).pin_memory(), torch.empty((P_POINTS, 4), dtype=torch.int32).pin_memory())
            for _ in range(S)]
    M = 0

    def e2e_run(nsteps):
        m = 0
        for i in range(nsteps + S - 1):     # software pipeline of depth S over the engine pool, one host thread
            if i < nsteps:
                engs[i % S].submit_host(pin[i % len(pin)], offs_pin, *outs[i % S])
            j = i - (S - 1)
            if j >= 0:
                m = engs[j % S].collect_host(*outs[j % S])
        torch.cuda.synchronize()
        return m

    M = e2e_run(2 * S)
    barrier()
    sampler.begin()
    t0 = time.perf_counter()
    M = e2e_run(args.steps)
    e2e_s = time.perf_counter() - t0
    sampler.end()
    clocks = sampler.stop()
    t = torch.tensor([e2e_s], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    e2e_value = world * args.steps / float(t.item())
    h2d = P_POINTS * eng.F * 4 + 8
    d2h = engs[0].d2h_rows * (eng.d * 4 + 16) + 4   # rows that actually crossed PCIe (predicted count >= M, see SSTEngine.submit_host)

    # ---- roofline of the dominant kernel group: the SRA encoder layers (attention + fused chain), timed as the 12-layer stack
    roof = None
    if rank == 0:
        import ctypes as C
        from sst_b200 import _lib as L
        feats, coors, num = step(0)
        torch.cuda.synchronize()
        Mv = int(num.item())
        d, ff = eng.d, cfg['backbone']['dim_feedforward'][0]
        flops_layers = []
        for sh in range(2):
            offs = eng.plans[sh]["win_offsets"]
            R = int(eng.plans[sh]["counters"][0].item())
            nw = (offs[1:R + 1] - offs[:R]).double()
            flops_layers.append(Mv * (8 * d * d + 4 * d * ff) + 4 * d * float((nw * nw).sum().item()))   # SURVEY.md 8d
        nl = len(eng._layers)
        flops = sum(flops_layers[l & 1] for l in range(nl)) / nl
        lib = L.lib()
        ts = []
        with torch.cuda.stream(st):
            c = L.ctx(dev)
            for it in range(10):
                flush.zero_()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(st)
                L.check(c, lib.sstb200_sra_stack_forward(c, eng._layer_array, nl, C.byref(eng._plan_structs[0]), C.byref(eng._plan_structs[1]),
                                                         eng.vf.data_ptr(), eng.x[0].data_ptr(), eng.x[1].data_ptr(), eng.cap,
                                                         eng.num.data_ptr(), {"fp32": 0, "bf16": 1}[precision]))
                b.record(st)
                ts.append((a, b))
        torch.cuda.synchronize()
        lt = sorted(x.elapsed_time(y) for x, y in ts[2:])
        layer_ms = lt[len(lt) // 2] / nl
        pk = peaks()
        ach = flops / (layer_ms * 1e-3) / 1e12
        traffic, traffic_src = None, None
        roof = {"bound": "tensor", "kernel": f"SRA encoder layer ({precision} path: window attention + wgmma GEMMs; average over the "
                                             f"{nl}-layer stack call, L2 flushed before the call)",
                "achieved": ach, "peak": pk["tf_sustained"], "unit": "TFLOP/s", "frac": ach / pk["tf_sustained"],
                "traffic": traffic, "traffic_source": traffic_src,
                "peak_source": pk["src"] + " bf16 dense",
                "flops_per_launch": flops, "ms_per_launch": layer_ms, "M": Mv,
                "layer_share_of_step": nl * layer_ms / latency_ms}

    # ---- fp32 (1e-3 tolerance) mode of the same workload, same protocol with fewer repetitions --------------------------
    fp32_rec = None
    if precision != "fp32" and not args.no_fp32:
        e32 = [SSTEngine(fl.VOXEL_SIZE, fl.PC_RANGE, vfe, il, bb, max_points=P_POINTS, batch_size=1, precision="fp32", device=dev)
               for _ in range(min(S, 4))]
        for i in range(len(e32) + 1):
            e32[i % len(e32)].load_frames_device(frames_d[i % NF], offs_d)
            e32[i % len(e32)].run()
        barrier()
        K32 = max(4, args.steps // 2)
        ws = []
        for rep in range(3):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(main)
            for e in e32:
                e.stream.wait_event(a)
            for i in range(K32):
                e = e32[i % len(e32)]
                e.load_frames_device(frames_d[(rep * K32 + i) % NF], offs_d)
                e.run()
            for e in e32:
                main.wait_stream(e.stream)
            b.record(main)
            ws.append((a, b))
        barrier()
        t32 = torch.tensor(sorted(a.elapsed_time(b) for a, b in ws), dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t32, op=dist.ReduceOp.MAX)
        ms32 = float(t32[len(ws) // 2])
        fp32_rec = {"value": world * K32 / (ms32 / 1e3), "unit": "frames/s", "steps": K32, "ms_per_step": ms32 / K32,
                    "frames_in_flight": len(e32), "tolerance": "1e-3 (fp32-tolerance mode, csrc/sra_fp32.cu: Linear layers as split-fp16 wgmma GEMMs with fp32 accumulation, fp32 SIMT window attention / LayerNorm)"}
        del e32

    # ---- training step (BASELINE config 4): fwd + bwd + ONE flat NCCL gradient all-reduce + fused AdamW, weak scaling ----
    train = None
    if not args.no_train:
        try:
            train = train_bench(args, world, rank, dev, frames_d)
        except Exception as e:   # the inference record must not be lost to a training-side failure; say so loudly instead
            train = {"error": f"{type(e).__name__}: {e}"}

    # ---- FSD sparse U-Net (SURVEY 8f next-1), single-GPU runs only (like the CPU baseline: no rank-0-only work between the
    # collectives of a multi-rank run and its process-group teardown): one sweep through SimpleSparseUNet, three precisions ----------
    fsd = None
    if rank == 0 and world == 1 and not args.no_fsd:
        try:
            fsd = fl.fsd_unet_bench(dev)
        except Exception as e:
            fsd = {"error": f"{type(e).__name__}: {e}"}

    sir = None
    if rank == 0 and world == 1 and not args.no_fsd:   # BASELINE config 3 beside it (same flag), never allowed to cost the main line
        try:
            sir = fl.sir_bench(dev)
        except Exception as e:
            sir = {"error": f"{type(e).__name__}: {e}"}

    cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        os.sched_setaffinity(0, all_cpus)   # the CPU baseline gets every host core again, like the --impl reference arm
        times, threads, _ = cpu_oracle_frames(6, 1, budget_s=30.0)
        cpu = {"value": len(times) / sum(times), "unit": "frames/s", "cores": threads, "kind": "port",
               "sample": f"{len(times)} frames of the same workload after 1 warm-up (oracle/sst_oracle.py, torch CPU fp32, "
                         f"{threads} threads)"}

    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": total_ms / args.steps, "windows": {"repeats": len(wms), "ms_min": wms[0], "ms_median": total_ms, "ms_max": wms[-1]},
            "latency_ms_single_stream": latency_ms, "value_one_frame_in_flight": world * 1e3 / latency_ms,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32" if precision == "fp32" else "f16", "data": "synthetic",
            "config": {"workload": WORKLOAD,
                       "precision": precision, "voxels": int(M), "frames_in_flight": S,
                       "host_cpus": (len(numa_cpus) if numa_cpus else None),
                       "l2": "inputs larger than L2: 80 distinct resident sweeps (144 MB) cycled; latency_ms measured with a 512 MB L2 flush per step",
                       "parallelism": f"dp{world} (frames sharded, no collective)"},
            "clocks": clocks, "gpu_launches": int(eng.launches_per_frame or 0) * args.steps,
            "gpu_graph_other_nodes_per_step": int(getattr(eng, "other_nodes_per_frame", 0) or 0),
            "gpu_launches_per_step": int(eng.launches_per_frame or 0),
            "e2e": {"value": e2e_value, "unit": "frames/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h},
            "roofline": roof, "cpu_baseline": cpu, "fp32": fp32_rec, "train": train, "fsd_unet": fsd, "fsd_sir": sir,
        }
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
