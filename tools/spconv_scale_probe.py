"""Per-row error of the three sparse-convolution precisions across operand scales, on the GPU.

    python tools/spconv_scale_probe.py [--rows 2000] [--out FILE.json]

One SubM 3x3x3 64 -> 64 convolution; features (then weights) multiplied by 2^s.  Printed per precision and s: the largest over output
rows of  |out[o] - ref[o]|_inf / |sum_k |x[nbr[o,k]]| @ |W[k]||_inf  with ref in float64 - the quantity tests/test_gpu_spconv_edges.py
bounds (fp32 1e-5, fp32_tc 1e-5, bf16 5e-3).  Power-of-two scaling is exact, so the columns of one precision should be equal.
One process, one launch per cell; the card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

S_FEATS = (-40, -30, -24, -20, -16, -12, -8, 0, 8, 14, 20, 30)
S_WEIGHT = (-30, -20, -12, -8, 0, 8, 14)


def reference(x, nbr, w):
    x, w = x.double(), w.double()
    acc = torch.zeros((nbr.shape[0], w.shape[2]), dtype=torch.float64)
    mag = torch.zeros_like(acc)
    for k in range(nbr.shape[1]):
        idx = nbr[:, k].long()
        m = idx >= 0
        acc[m] += x[idx[m]] @ w[k]
        mag[m] += x[idx[m]].abs() @ w[k].abs()
    return acc, mag.amax(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from oracle import spconv_oracle as SO
    from sst_b200 import spconv_modules as SP
    dev = torch.device("cuda:0")
    shape = [10, 40, 40]
    feats, coors = SO.synth_sparse(1, 2, shape, a.rows // 2, 64)
    w = torch.randn((27, 64, 64), generator=torch.Generator().manual_seed(2)) / (27 * 64) ** 0.5 * 2
    nbr, _ = SP.conv_table(coors.to(dev), coors.to(dev), 2, shape, shape, [3, 3, 3], [1, 1, 1], [1, 1, 1])
    ref, bound = reference(feats, nbr.cpu(), w)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(card=card, rows=int(coors.shape[0]), features={}, weights={})
    for key, scales in (("features", S_FEATS), ("weights", S_WEIGHT)):
        for prec in ("fp32", "bf16", "fp32_tc"):
            row = {}
            for s in scales:
                f = 2.0 ** s
                out = SP.indice_conv((feats * f if key == "features" else feats).to(dev), nbr,
                                     (w * f if key == "weights" else w).to(dev), precision=prec).double().cpu()
                row[s] = float(((out - ref * f).abs().amax(1) / (bound * f)).max())
            res[key][prec] = row
            print(f"{key:8s} {prec:7s} " + "  ".join(f"2^{s}: {v:.1e}" for s, v in row.items()))
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
