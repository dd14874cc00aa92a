"""Step time of TrainStep (bf16 training path) with plain and with cosine attention, in one process.

Both models are the flagship SST (6 blocks, d 128, 8 heads) and differ only in layer_cfg: cosine=True, tau_min=0.01 for the second.
Each timed round runs `--steps` steps of one variant, then of the other, alternating for `--rounds` rounds, after `--warmup` steps
of each.  Times come from CUDA events around each round; the card's name and power limit are printed beside them.

    python tools/train_step_timing.py [--frames 4] [--points 150000] [--steps 5] [--rounds 4] [--warmup 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from sst_b200 import flagship as fl  # noqa: E402
from sst_b200.train import TrainStep  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return name, q or "unknown"


def make_step(cosine, dev):
    cfg = fl.sst_cfg()
    cfg["backbone"]["precision"] = "bf16"
    if cosine:
        cfg["backbone"]["layer_cfg"] = dict(cosine=True, tau_min=0.01)
    vfe, il, bb = fl.build_sst(cfg)
    return TrainStep(vfe.to(dev), il, bb.to(dev), fl.VOXEL_SIZE, fl.PC_RANGE)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--points", type=int, default=150000)
    ap.add_argument("--steps", type=int, default=5, help="steps per timed round")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("train_step_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    frames = [fl.synth_frame(1000 + i, a.points).to(dev) for i in range(a.frames)]
    steps = {"plain": make_step(False, dev), "cosine": make_step(True, dev)}
    for ts in steps.values():
        for _ in range(a.warmup):
            ts.step(frames)
    torch.cuda.synchronize()
    ms = {k: [] for k in steps}
    for _ in range(a.rounds):
        for k, ts in steps.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                ts.step(frames)
            e1.record()
            e1.synchronize()
            ms[k].append(e0.elapsed_time(e1) / a.steps)
    name, power = card()
    res = {"gpu": name, "power_limit": power, "frames": a.frames, "points_per_frame": a.points, "steps_per_round": a.steps,
           "rounds": a.rounds}
    for k, v in ms.items():
        res[f"{k}_ms_per_step_median"] = round(statistics.median(v), 3)
        res[f"{k}_ms_per_step_rounds"] = [round(x, 3) for x in v]
    res["cosine_over_plain"] = round(res["cosine_ms_per_step_median"] / res["plain_ms_per_step_median"], 4)
    print(f"{name}, power limit {power}: {a.frames} x {a.points} points, median step plain {res['plain_ms_per_step_median']:.2f} ms, "
          f"cosine {res['cosine_ms_per_step_median']:.2f} ms")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
