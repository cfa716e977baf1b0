"""The UNMODIFIED reference's Net.step(batch, "train") plus backward and Net.step_inference(batch, "test") on the drop-in,
with the decoder hook off and on (pasco_b200/hooks.py install(decoder=True)); the attention, post-processing, evaluation,
criterion and trunk hooks are on in both arms.

    python tools/decoder_hook_bench.py [--train 1 2] [--test 1 3] [--steps 6] [--warmup 1]

Workload: tools/criterion_hook_bench.py's training batch and tools/evaluate_hook_bench.py's test batch at 256x256x32
@10 % (f = 64, Q = 100), decoder off and on alternated step by step.  Per arm:
  * the step's median and range in ms (host clock, ended by a device synchronise);
  * the forward time inside each hooked function (DecoderGenerativeSepConvV2.forward and, inside it, the four
    DecoderBlock.forward calls, predict_completion_sem_logit and predict_panop), every call bracketed by device
    synchronises, in a separate pass; "decoder_share" is the whole decoder forward's median over the step's median;
  * host synchronisations (torch.cuda.set_sync_debug_mode), kernel launches (torch.profiler) and peak memory.
Prints one JSON line per workload, with the card's name, power limit and SM clock read in the same run; writes nothing.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle", "_ref"), os.path.join(ROOT, "compat"),
                os.path.join(ROOT, "tests", "golden")]
from evaluate_hook_bench import counted, fresh_metrics, stats, timed, with_gt  # noqa: E402
from infer_bench import GRID  # noqa: E402
from postprocess_bench import batch_of, calibrate, reference_net  # noqa: E402
import trunk_hook_bench as TB  # noqa: E402

TB.HOOKED = (("pasco.models.decoder_v3", "DecoderGenerativeSepConvV2", "forward"),
             ("pasco.models.decoder_v3", "DecoderBlock", "forward"),
             ("pasco.models.decoder_v3", "DecoderGenerativeSepConvV2", "predict_completion_sem_logit"),
             ("pasco.models.decoder_v3", "DecoderGenerativeSepConvV2", "predict_panop"))


def set_hooks(hooks, on):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=True, evaluate=True, criterion=True, trunk=True, decoder=on)


def alternate(one, hooks, a):
    times = {False: [], True: []}
    for i in range(a.warmup + a.steps):
        for on in (False, True) if i % 2 == 0 else (True, False):
            set_hooks(hooks, on)
            t = timed(one)
            if i >= a.warmup:
                times[on].append(t)
    out = {}
    for on in (False, True):
        set_hooks(hooks, on)
        arm = dict(stats(times[on]), **TB.hooked_time(one, 3), **counted(one))
        fwd = arm.get("DecoderGenerativeSepConvV2.forward_ms")
        if fwd is not None:
            arm["decoder_share"] = round(fwd / arm["ms_median"], 3)
        out["decoder_on" if on else "decoder_off"] = arm
    hooks.uninstall()
    return out


def train(M, a, hooks, make_scene):
    from dropin_scale_bench import train_batch
    net = reference_net(M).train()
    K = net.n_classes
    net.class_weights = [torch.ones(K + 1) for _ in range(M)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K, device="cuda")
    net.object_mask_threshold = 0.05
    net.log = lambda *x, **k: None
    batch = train_batch(make_scene, M, 0)

    def one():
        torch.manual_seed(0)
        net.zero_grad(set_to_none=True)
        net.step(batch, "train")["loss"].backward()

    out = {"workload": f"Net.step(batch, 'train') + backward, M = {M}, {'x'.join(map(str, GRID))} @10 %",
           "steps": a.steps, "gpu": TB.gpu_state(), **alternate(one, hooks, a)}
    del net, batch
    torch.cuda.empty_cache()
    return out


def test(M, a, hooks, make_scene):
    net = reference_net(M)
    batch = with_gt(make_scene, batch_of(make_scene, M, 1), M, 1)
    set_hooks(hooks, False)
    calibrate(net, batch)
    net.object_mask_threshold = 0.05
    net.log = lambda *x, **k: None

    def one():
        fresh_metrics(net)
        torch.manual_seed(0)
        with torch.no_grad():
            net.step_inference(batch, "test", eval=True)

    out = {"workload": f"Net.step_inference(batch, 'test'), M = {M}, {'x'.join(map(str, GRID))} @10 %",
           "steps": a.steps, "gpu": TB.gpu_state(), **alternate(one, hooks, a)}
    del net, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train", type=int, nargs="*", default=[1, 2])
    ap.add_argument("--test", type=int, nargs="*", default=[1, 3])
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decoder_hook_bench.py: no CUDA device")
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "pasco")):
        raise SystemExit("decoder_hook_bench.py: the reference is not staged under oracle/_ref (run build())")
    from pasco_b200 import _lib, hooks, ops
    _lib.load()
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    for M in a.train:
        print(json.dumps(train(M, a, hooks, make_scene)), flush=True)
    for M in a.test:
        print(json.dumps(test(M, a, hooks, make_scene)), flush=True)


if __name__ == "__main__":
    main()
