"""The UNMODIFIED reference's Net.step(batch, "train") plus backward and Net.step_inference(batch, "test") on the drop-in,
with the transformer hook off and on (pasco_b200/hooks.py install(transformer=True)); the attention, post-processing,
evaluation, criterion, trunk and decoder hooks are on in both arms.

    python tools/transformer_hook_bench.py [--train 1 2] [--test 1 3] [--steps 6] [--warmup 1] [--profile]

Workload: tools/decoder_hook_bench.py's training and test batches at 256x256x32 @10 % (f = 64, Q = 100), transformer
off and on alternated step by step.  Per arm:
  * the step's median and range in ms (host clock, ended by a device synchronise);
  * the time inside TransformerPredictorV2.forward, every call bracketed by device synchronises, in a separate pass;
  * host synchronisations (torch.cuda.set_sync_debug_mode), kernel launches (torch.profiler) and peak memory.
--profile: instead, one torch.profiler run of the M = 1 test step per arm, with the device time of every kernel inside
TransformerPredictorV2.forward given to the piece of the forward it ran in (ranges around the reference's submodules
and the hooks' helpers; element-wise add kernels in the cross-attention layers and outside every range are the
`+ pos` passes).  Prints one JSON line per workload or arm, with the card's name, power limit and SM clock read in the
same run; writes nothing.
"""
import argparse
import collections
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

TB.HOOKED = (("pasco.models.transformer.transformer_predictor_v2", "TransformerPredictorV2", "forward"),)


def set_hooks(hooks, on):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=True, evaluate=True, criterion=True, trunk=True, decoder=True,
                         transformer=on)


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
        out["transformer_on" if on else "transformer_off"] = dict(stats(times[on]), **TB.hooked_time(one, 3),
                                                                  **counted(one))
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


def inference_setup(M, hooks, make_scene):
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
    return net, batch, one


def test(M, a, hooks, make_scene):
    net, batch, one = inference_setup(M, hooks, make_scene)
    out = {"workload": f"Net.step_inference(batch, 'test'), M = {M}, {'x'.join(map(str, GRID))} @10 %",
           "steps": a.steps, "gpu": TB.gpu_state(), **alternate(one, hooks, a)}
    del net, batch
    torch.cuda.empty_cache()
    return out


# ------------------------------------------------------------------------------------------------
# --profile: device time per piece of TransformerPredictorV2.forward
# ------------------------------------------------------------------------------------------------
def _ranged(label, fn):
    def inner(*a, **k):
        with torch.profiler.record_function(label):
            return fn(*a, **k)
    return inner


def _pieces(tp, hooks):
    """Put a profiler range around every piece of the forward; returns the undo list."""
    undo = []

    def on_obj(obj, name, label):
        undo.append((obj, name, obj.__dict__.get(name)))
        setattr(obj, name, _ranged(label, getattr(obj, name)))

    def pe_call(fn):
        def inner(*a, **k):
            with torch.profiler.record_function(next(pe_labels)):
                return fn(*a, **k)
        return inner
    pe_labels = iter([f"tf:pe_layer s{s}" for _ in range(1000) for s in tp.src_scales])
    undo.append((tp.pe_layer, "forward", tp.pe_layer.__dict__.get("forward")))
    tp.pe_layer.forward = pe_call(tp.pe_layer.forward)
    on_obj(tp.mask_feat_proj, "forward", "tf:projections")
    for m in tp.input_projs:
        on_obj(m, "forward", "tf:projections")
    on_obj(tp, "pred_heads", "tf:pred_heads (mask head einsums)")
    for m in tp.transformer_cross_attention_layers:
        on_obj(m, "forward", "tf:cross-attention")
    for m in list(tp.transformer_self_attention_layers) + list(tp.transformer_ffn_layers):
        on_obj(m, "forward", "tf:self-attention + FFN")
    for name, label in (("_mask_bits", "tf:mask bits"), ("_voxel_map", "tf:mask bits"),
                        ("_proj_plus_pos", "tf:projections + pos (proj_plus_pos)"),
                        ("_item_outputs", "tf:per-item outputs")):
        undo.append((hooks, name, getattr(hooks, name)))
        setattr(hooks, name, _ranged(label, getattr(hooks, name)))
    return undo


def _attribute(prof):
    """ms of device time per piece: each kernel goes to the innermost profiler range whose device span holds it."""
    evs = prof.events()
    cuda = torch.autograd.DeviceType.CUDA
    spans = [(e.time_range.start, e.time_range.end, e.name) for e in evs
             if e.device_type == cuda and e.name.startswith("tf:")]
    kernels = [e for e in evs if e.device_type == cuda and not e.name.startswith("tf:")
               and not e.name.startswith(("Memcpy", "Memset"))]
    out = collections.defaultdict(float)
    for k in kernels:
        t = k.time_range.start
        inside = [s for s in spans if s[0] <= t < s[1]]
        if not inside:
            continue
        label = min(inside, key=lambda s: s[1] - s[0])[2]
        is_add = "add" in k.name.lower() and "elementwise" in k.name.lower()
        if label == "tf:forward":
            label = "+ pos adds (outside the submodules)" if is_add else "rest (per-item outputs, reshapes, stacks)"
        elif label == "tf:cross-attention" and is_add:
            label = "+ pos adds (in the cross-attention layers)"
        elif label == "tf:projections + pos (proj_plus_pos)":
            label = "+ pos (ops.sine_pos add pass)" if "sine_pos" in k.name else "projections"
        out[label.replace("tf:", "")] += k.time_range.elapsed_us() / 1e3
    return {k: round(v, 2) for k, v in sorted(out.items(), key=lambda kv: -kv[1])}


def profile(hooks, make_scene):
    from torch.profiler import ProfilerActivity, profile as prof_ctx
    from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    net, batch, one = inference_setup(1, hooks, make_scene)
    tp = net.unet3d.decoder_generative.transformer_predictor
    rows = []
    for on in (False, True):
        set_hooks(hooks, on)
        one()
        undo = _pieces(tp, hooks)
        fwd = TransformerPredictorV2.forward
        TransformerPredictorV2.forward = _ranged("tf:forward", fwd)
        try:
            torch.cuda.synchronize()
            with prof_ctx(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
                one()
                torch.cuda.synchronize()
        finally:
            TransformerPredictorV2.forward = fwd
            for obj, name, old in undo:
                if old is None and isinstance(obj, torch.nn.Module):
                    delattr(obj, name)
                else:
                    setattr(obj, name, old)
        pieces = _attribute(p)
        rows.append({"arm": "transformer_on" if on else "transformer_off", "gpu": TB.gpu_state(),
                     "kernel_ms_by_piece": pieces, "kernel_ms_sum": round(sum(pieces.values()), 2)})
    hooks.uninstall()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train", type=int, nargs="*", default=[1, 2])
    ap.add_argument("--test", type=int, nargs="*", default=[1, 3])
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transformer_hook_bench.py: no CUDA device")
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "pasco")):
        raise SystemExit("transformer_hook_bench.py: the reference is not staged under oracle/_ref (run build())")
    from pasco_b200 import _lib, hooks, ops
    _lib.load()
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    if a.profile:
        for row in profile(hooks, make_scene):
            print(json.dumps(row), flush=True)
        return
    for M in a.train:
        print(json.dumps(train(M, a, hooks, make_scene)), flush=True)
    for M in a.test:
        print(json.dumps(test(M, a, hooks, make_scene)), flush=True)


if __name__ == "__main__":
    main()
