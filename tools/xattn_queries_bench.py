"""Times the masked cross-attention entry points (pasco_xattn_forward / pasco_xattn_backward) against the query count.

    python tools/xattn_queries_bench.py [--root TREE] [--queries 100 128 200 256] [--keys 25000 120000 400000]

For every (P keys, Q queries) at H = 8 heads of width 48 (the network's shape) with a random mask of about a quarter
of the keys: median and spread of 30 timed calls after 5 warm-ups, CUDA events around each call.  Prints one JSON line
per shape, with the pool workspace each call takes (the same sizes xattn.cu's xattn_setup allocates).  `--root` imports
the library of another tree (e.g. a parent checkout) to alternate two builds in one session.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys


def workspace_bytes(P, Q, H, D, sms):
    """bytes the forward / backward take from the library's pool (xattn.cu pick_chunks / xattn_setup)"""
    nqb = (Q + 127) // 128
    chunks = max(1, min((P + 63) // 64, -(-sms // (H * nqb))))
    part = chunks * Q * H * D
    return 4 * (part + chunks * H * Q * 2), 4 * (part + (nqb - 1) * 2 * P * H * D)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--queries", type=int, nargs="+", default=[100, 128, 200, 256])
    ap.add_argument("--keys", type=int, nargs="+", default=[25_000, 120_000, 400_000])
    ap.add_argument("--heads", type=int, default=8)
    ap.add_argument("--dim", type=int, default=48)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--tag", default="")
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.root))
    import torch
    from pasco_b200 import ops
    from pasco_b200._lib import ptr
    if not torch.cuda.is_available():
        sys.exit("xattn_queries_bench: needs a CUDA device")
    dev = torch.device("cuda")
    props = torch.cuda.get_device_properties(0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": props.name, "power_limit_and_max_sm_clock": smi[0] if smi else "unknown",
                      "lib": os.path.abspath(ops.__file__), "tag": a.tag}), flush=True)
    H, D = a.heads, a.dim
    HD, scale = H * D, C.c_float(D ** -0.5)
    g = torch.Generator(device=dev).manual_seed(0)
    for P in a.keys:
        k = torch.randn(P, HD, device=dev, generator=g)
        v = torch.randn(P, HD, device=dev, generator=g)
        dk, dv = torch.empty_like(k), torch.empty_like(v)
        for Q in a.queries:
            q = torch.randn(Q, HD, device=dev, generator=g)
            go = torch.randn(Q, HD, device=dev, generator=g)
            W = 2 * ((P + 63) // 64)
            bits = (torch.randint(0, 2 ** 31, (Q, W), device=dev, generator=g, dtype=torch.int64)
                    & torch.randint(0, 2 ** 31, (Q, W), device=dev, generator=g, dtype=torch.int64)).to(torch.int32)
            out, lse, dq = torch.empty(Q, HD, device=dev), torch.empty(H, Q, device=dev), torch.empty(Q, HD, device=dev)

            def fwd():
                ops.call("pasco_xattn_forward", ptr(q), ptr(k), ptr(v), ptr(bits), Q, P, H, D, scale, ptr(out), ptr(lse))

            def bwd():
                ops.call("pasco_xattn_backward", ptr(q), ptr(k), ptr(v), ptr(bits), ptr(lse), ptr(out), ptr(go), Q, P,
                         H, D, scale, ptr(dq), ptr(dk), ptr(dv))

            res = {"P": P, "Q": Q, "H": H, "D": D, "tag": a.tag}
            try:
                fwd()
                torch.cuda.synchronize()
            except RuntimeError as e:                   # a build without query blocks rejects Q > 128
                res["error"] = str(e)[:120]
                print(json.dumps(res), flush=True)
                continue
            for name, fn in (("fwd", fwd), ("bwd", bwd)):
                for _ in range(a.warmup):
                    fn()
                ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(a.iters)]
                for e0, e1 in ev:
                    e0.record()
                    fn()
                    e1.record()
                torch.cuda.synchronize()
                ts = sorted(e0.elapsed_time(e1) for e0, e1 in ev)
                res[f"{name}_ms"] = round(statistics.median(ts), 4)
                res[f"{name}_ms_min_max"] = [round(ts[0], 4), round(ts[-1], 4)]
            res["ws_fwd_bytes"], res["ws_bwd_bytes"] = workspace_bytes(P, Q, H, D, props.multi_processor_count)
            print(json.dumps(res), flush=True)
            del q, go, bits, out, lse, dq
        del k, v, dk, dv
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
