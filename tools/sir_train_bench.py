"""CUDA-event timing of SIR training: the native fp32 SirLayerFunction (csrc/sir.cu forward with state + csrc/sir_train.cu backward)
against SIRLayer._forward_composed (torch Linear / LayerNorm / activation around ops.segment_reduce, autograd) on the same GPU tensors.
Workloads: config-3 SIR (3 blocks, 84/133/133, [128, 128], rel [16, 32], GELU; 150k points, 256 groups) and FullySparseBboxHead's
stack of 6 SIRLayers (in 213 then 146, rel_in 13, [128, 128]; 100k pooled points over 1000 RoIs).  For each side: forward + backward
(median of 3 alternating rounds), the backward alone with achieved FLOP/s from the count below, the bytes held for the backward
(memory_allocated after the forward minus before), and the largest relative difference between the two sides' outputs and gradients.
Prints the card name and power limit read in the same run; writes OUT/sir_train_bench.json.
`python tools/sir_train_bench.py [--iters K] [--out DIR]`"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return name, q or "unknown"


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def layer_bwd_flops(N, G, cin, C0, C1, rel_in, rel_dims):
    """Multiply-adds x 2 of one SIRLayer backward as sir_train.cu runs it: dW0, dx0, dW1a, dp0, S1 W1b, dW1b, and the rel-MLP
    (forward recompute, input gradient and weight gradient of each layer, plus the x0 recompute)."""
    f = 2 * N * C0 * cin * 2
    if C1:
        f += 2 * N * C1 * C0 * 2 + 2 * G * C1 * C0 * 2
    ins = [rel_in] + rel_dims[:-1]
    f += 2 * N * sum(i * o for i, o in zip(ins, rel_dims)) * 4
    return f


def sync_grads(m):
    for p in m.parameters():
        p.grad = None


def composed(m):
    from sst_b200.sir_modules import SIRLayer
    for blk in m.modules():
        if isinstance(blk, SIRLayer):
            blk._native_train = lambda: False


def config3(dev, native):
    from sst_b200.sir_modules import SIR
    torch.manual_seed(0)
    m = SIR(num_blocks=3, in_channels=[84, 133, 133], feat_channels=[[128, 128]] * 3, rel_mlp_hidden_dims=[[16, 32]] * 3,
            norm_cfg=dict(type='LN', eps=1e-3), mode='max', xyz_normalizer=[20, 20, 4], act='gelu', unique_once=True).to(dev).train()
    if not native:
        composed(m)
    N, G = 150000, 256
    g = torch.Generator().manual_seed(1)
    points = torch.cat([torch.randn(N, 3, generator=g) * 10, torch.rand(N, 2, generator=g)], 1).to(dev)
    feats = torch.randn(N, 79, generator=g).to(dev).requires_grad_(True)
    gid = torch.randint(0, G, (N,), generator=g)
    coors = torch.stack([gid % 3, torch.zeros_like(gid), gid], 1).to(dev)
    fcl = (torch.randn(N, 3, generator=g) * 2).to(dev)
    probes = [torch.randn(N, 128, generator=g).to(dev), torch.randn(G, 768, generator=g).to(dev)]

    def fwd():
        a, b, _ = m(points, feats, coors, fcl)
        return [a, b]
    flops = sum(layer_bwd_flops(N, G, cin, 128, 128, 3, [16, 32, cin]) for cin in (84, 133, 133))
    return m, fwd, probes, [feats], flops


def roi_head(dev, native):
    from sst_b200 import ops
    from sst_b200.sir_modules import SIRLayer
    torch.manual_seed(0)
    ins = [213] + [146] * 5
    layers = torch.nn.ModuleList([SIRLayer(in_channels=c, feat_channels=[128, 128], rel_mlp_hidden_dims=[16, 32], rel_mlp_in_channel=13,
                                           norm_cfg=dict(type='LN', eps=1e-3), mode='max', return_point_feats=True, rel_dist_scaler=10.0,
                                           xyz_normalizer=[20, 20, 4], act='gelu') for c in ins]).to(dev).train()
    if not native:
        composed(layers)
    N, R = 100000, 1000
    g = torch.Generator().manual_seed(2)
    x = torch.randn(N, 213, generator=g).to(dev).requires_grad_(True)
    rid = torch.sort(torch.randint(0, R, (N,), generator=g)).values
    coors = torch.stack([torch.zeros_like(rid), rid], 1).to(dev)
    fcl = (torch.randn(N, 13, generator=g) * 2).to(dev)
    new_coors, inv = ops.unique_rows(coors)
    probes = [torch.randn(N, 128, generator=g).to(dev), torch.randn(R, 256 * 6, generator=g).to(dev)]

    def fwd():
        h, gl = x, []
        for i, l in enumerate(layers):
            pf, gf = l(h, coors, fcl, unq_inv_once=inv, new_coors_once=new_coors)
            gl.append(gf)
            h = torch.cat([x[:, :18], pf], 1)
        return [pf, torch.cat(gl, 1)]
    flops = sum(layer_bwd_flops(N, R, c, 128, 128, 13, [16, 32, c]) for c in ins)
    return layers, fwd, probes, [x], flops


def run(build, dev, iters):
    sides = {}
    for native in (True, False):
        m, fwd, probes, leaves, flops = build(dev, native)
        sides[native] = dict(m=m, fwd=fwd, probes=probes, leaves=leaves, flops=flops)

    def step(s):
        outs = s["fwd"]()
        torch.autograd.backward(outs, s["probes"])
        for t in s["leaves"]:
            t.grad = None
        sync_grads(s["m"])
    res = {}
    rounds = {True: [], False: []}
    for _ in range(3):  # alternate the two sides in one process
        for native in (True, False):
            rounds[native].append(timed(lambda: step(sides[native]), iters))
    for native in (True, False):
        s = sides[native]
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        outs = s["fwd"]()
        torch.cuda.synchronize()
        held = torch.cuda.memory_allocated() - before

        def bwd():
            torch.autograd.backward(outs, s["probes"], retain_graph=True)
        t_bwd = timed(bwd, iters)
        for t in s["leaves"]:
            t.grad = None
        sync_grads(s["m"])
        torch.autograd.backward(outs, s["probes"])
        s["result"] = [o.detach() for o in outs] + [t.grad for t in s["leaves"]] + [p.grad for p in s["m"].parameters()]
        del outs
        res["native" if native else "composed"] = dict(
            fwd_bwd_ms=statistics.median(rounds[native]), bwd_ms=t_bwd, bwd_tflops=(s["flops"] / (t_bwd * 1e-3) / 1e12) if native else None,
            bytes_held_for_backward=held)
    diff = 0.0
    for a, b in zip(sides[True]["result"], sides[False]["result"]):
        diff = max(diff, (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30))
    res["max_rel_diff_native_vs_composed"] = diff
    res["speedup_fwd_bwd"] = res["composed"]["fwd_bwd_ms"] / res["native"]["fwd_bwd_ms"]
    res["bwd_flop_count"] = sides[True]["flops"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default="sir_train_bench_out")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    name, power = card()
    print(f"card: {name}; power limit, max SM clock: {power}")
    out = dict(card=name, power_limit_and_max_sm_clock=power, iters=args.iters)
    for key, build in (("config3_sir_150k_256", config3), ("roi_head_6_layers_100k_1000", roi_head)):
        out[key] = run(build, dev, args.iters)
        print(key, json.dumps(out[key], indent=1))
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "sir_train_bench.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
