"""Micro-benchmark of the map-building and convolution kernels on BASELINE-shaped synthetic scenes.

    python tools/conv_microbench.py [--occ 0.1] [--channels 64] [--stride 1] [--out FILE.jsonl]

--stride S times the level-S coordinate set of the same synthetic grid (coordinates divided by S, duplicates merged),
so that a kernel runs at the size it has at the network's stride-S level: the network convolves 64 channels at stride
1, 128 at stride 2 and 256 at strides 4 and 8.

Times each kernel with CUDA events (3 warm-ups, 10 timed launches, L2 flushed between launches by
writing a 256 MB buffer) and prints achieved algorithmic GB/s / TFLOP/s per SURVEY.md §8d formulas.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pasco_b200 import build  # noqa: E402

build.build()
from pasco_b200 import me as ME, ops  # noqa: E402


def timed(fn, iters=10, warm=3, flush=None):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, nargs=3, default=[256, 256, 32])
    ap.add_argument("--occ", type=float, nargs="+", default=[0.1, 0.5])
    ap.add_argument("--channels", type=int, nargs="+", default=[64, 128])
    ap.add_argument("--stride", type=int, default=1)
    ap.add_argument("--out", default="gpurun_out/micro.jsonl")
    a = ap.parse_args()
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = open(a.out, "a")

    def emit(**kw):
        print(json.dumps(kw))
        out.write(json.dumps(kw) + "\n")
        out.flush()

    for occ in a.occ:
        g = torch.Generator(device="cpu").manual_seed(0)
        o = torch.rand(*a.grid, generator=g) < occ
        c = torch.nonzero(o).int()
        if a.stride > 1:
            c = torch.unique(torch.div(c, a.stride, rounding_mode="floor"), dim=0)
        C = torch.cat([torch.zeros(c.shape[0], 1, dtype=torch.int32), c], 1).to(dev)
        N = C.shape[0]
        t_ins = timed(lambda: ops.hash_insert(C), flush=flush)
        table, _ = ops.hash_insert(C)
        t_probe = timed(lambda: ops.kernel_map_probe(C, table, 3, (1, 1, 1)), flush=flush)
        nbr = ops.kernel_map_probe(C, table, 3, (1, 1, 1))
        pairs = int((nbr >= 0).sum())
        emit(kind="maps", occ=occ, stride=a.stride, N=N, pairs=pairs, insert_ms=t_ins, probe_ms=t_probe,
             insert_GBs=16 * N / t_ins / 1e6, probe_GBs=(16 + 4 * 27) * N / t_probe / 1e6)
        for ch in a.channels:
            F = torch.randn(N, ch, device=dev)
            W = torch.randn(27, ch, ch, device=dev) * 0.05
            G = torch.randn(N, ch, device=dev)
            pk = ops.PackedWeights()
            koff = [26 - k for k in range(27)]
            for prec in ("fp32", "bf16"):
                ops.set_precision(prec)
                ops.use_planes(True)
                split = timed(lambda: ops.split_planes(F), flush=flush)
                fp, gp = ops.split_planes(F), ops.split_planes(G)
                fwd_pl = timed(lambda: ops.conv_apply(F, W, nbr, N, False, None, packs=pk, planes=fp), flush=flush)
                dgr_pl = timed(lambda: ops.conv_apply(G, W, nbr, N, True, koff, packs=pk, planes=gp), flush=flush)
                wgr_pl = timed(lambda: ops.conv_wgrad(F, G, nbr, 27, ch, ch, in_planes=fp, g_planes=gp), flush=flush)
                ops.use_planes(False)
                fwd = timed(lambda: ops.conv_apply(F, W, nbr, N, False, None, packs=pk), flush=flush)
                dgr = timed(lambda: ops.conv_apply(G, W, nbr, N, True, koff, packs=pk), flush=flush)
                wgr = timed(lambda: ops.conv_wgrad(F, G, nbr, 27, ch, ch), flush=flush)
                ops.use_planes(True)
                flops = 2.0 * pairs * ch * ch
                issued = 2.0 * N * 27 * ch * ch * (3 if prec == "fp32" else 1)
                bytes_min = 4.0 * (2 * N * ch) + 4.0 * 27 * ch * ch + 8.0 * pairs
                emit(kind="conv3", occ=occ, stride=a.stride, N=N, C=ch, pairs=pairs, precision=prec, split_ms=split,
                     fwd_planes_ms=fwd_pl, dgrad_planes_ms=dgr_pl, wgrad_planes_ms=wgr_pl,
                     fwd_regs_ms=fwd, dgrad_regs_ms=dgr, wgrad_regs_ms=wgr,
                     fwd_planes_useful_TFLOPs=flops / fwd_pl / 1e9, fwd_planes_issued_TFLOPs=issued / fwd_pl / 1e9,
                     wgrad_planes_useful_TFLOPs=flops / wgr_pl / 1e9, wgrad_planes_issued_TFLOPs=issued / wgr_pl / 1e9,
                     fwd_planes_alg_GBs=bytes_min / fwd_pl / 1e6, wgrad_planes_alg_GBs=bytes_min / wgr_pl / 1e6,
                     gather_GBs=pairs * ch * (4 if prec == "fp32" else 2) / fwd_pl / 1e6)
            ops.set_precision("fp32")
            if N <= 300000 and ch == 64:
                ops.force_simt(True)
                simt = timed(lambda: ops.conv_apply(F, W, nbr, N, False, None), iters=3, warm=1)
                ops.force_simt(False)
                emit(kind="conv3_simt", occ=occ, N=N, C=ch, fwd_ms=simt)


if __name__ == "__main__":
    main()
