#!/usr/bin/env python
"""Generate tests/golden/* by RUNNING THE REFERENCE (jakc4103/DFQ, imported unmodified from /root/reference) in the
build container.  Committed next to its outputs so every fixture can be regenerated.

  topology_<model>.json   node types / layer hyper-parameters / edges of the reference's own trace (PyTransformer) of
                          MobileNetV2, ResNet-18, DeepLab-v3+ (MobileNetV2) and MobileNetV2-SSD-lite with ReLU6 -> ReLU
  ref_<model>.npz         results of the reference's merge_batchnorm -> create_relation -> cross_layer_equalization
                          -> bias_correction (-> quantize_targ_layer) on the seeded random model that
                          dfq_b200.workload.build_graph materialises from the topology: relation lists, sweep counts,
                          every S / bias / fake_weight / fake_bias vector, and per-layer weight digests
                          (sha256 + max|w| + fp64 sum) after each stage
  ref_ops.npz             op-level vectors: _layer_equalization on the shapes of Appendix B, UniformQuantize codes,
                          QuantMeasure updates, _quantize_error

  ref_bc_<model>.npz      the reference's dfq.bias_correction ALONE on seed-regenerable inputs (tests/bc_fixture.py):
                          every post-correction bias and fake_bias vector + sha256 of every input tensor
  main_<cls|seg|ssd>.npz  made by tests/main_harness.py --impl reference (the unmodified main scripts end to end)

  ref_live_pins.npz       the reference's _layer_equalization, replace_op forward and getDistilData on the inputs of the
                          pin tests (tests/test_oracle_pins.py, test_op_patching.py, test_distill.py)

  ref_ssd_postprocess.npz the reference's Predictor.predict post-processing on seeded SSD-Lite-shaped outputs
  ref_ssd_soft_nms.npz    the same with Predictor(nms_method="soft"): soft_nms on the CPU, sigma 0.3, top_k -1 / 1 / 5
  ref_seg_eval.npz        the reference's forward_all predictions and Evaluator matrices and metrics on seeded batches
  ref_ssd_map.npz         main_ssd.py's per-class VOC average precision on a seeded set of detections and annotations
  ref_absorb_clip.npz     the reference's merge_batchnorm -> cross_layer_equalization -> bias_absorption -> clip_weight ->
                          bias_correction (main_cls.py:149-181 with --relu --equalize --absorption --clip_weight
                          --correction) on the seeded models of tests/absorb_clip_case.py: every weight, bias,
                          fake_bias after equalization, after absorption, after the clip and at the end (weights: after
                          equalization and after the clip)

usage: python tools/make_golden.py [topology] [mobilenetv2] [resnet18] [deeplab] [ssd] [ops] [bc] [minmax] [table] [live]
       [ssd_post] [ssd_soft] [seg_eval] [ssd_map] [absorb_clip]
"""
import hashlib
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

import refenv  # noqa: E402

ref = refenv.install()
os.chdir(refenv.REF_ROOT)
from dfq_b200 import workload  # noqa: E402  (pure python/torch; builds the seeded graphs)


def digest(t: torch.Tensor):
    a = np.ascontiguousarray(t.detach().cpu().numpy())
    return hashlib.sha256(a.tobytes()).hexdigest(), float(np.abs(a).max()), float(a.astype(np.float64).sum())


# ---------------------------------------------------------------------------------------------------------
def trace_topology(name):
    TT = refenv.tracer()
    if name == "mobilenetv2":
        from modeling.classification.MobileNetV2 import mobilenet_v2
        model, data = mobilenet_v2(None), torch.ones((4, 3, 224, 224))
    elif name == "resnet18":
        import torchvision.models as models
        model, data = models.resnet18(), torch.ones((4, 3, 224, 224))
    elif name == "deeplab":
        from modeling.segmentation.deeplab import DeepLab
        model, data = DeepLab(sync_bn=False), torch.ones((4, 3, 513, 513))
    elif name == "ssd":
        from modeling.detection.mobilenet_v2_ssd_lite import create_mobilenetv2_ssd_lite
        model, data = create_mobilenetv2_ssd_lite(21, width_mult=1.0), torch.ones((4, 3, 300, 300))
    else:
        raise ValueError(name)
    model.eval()
    tr = TT()
    model, tr = ref.layer_transform.switch_layers(model, tr, data, {0: [(nn.ReLU6, nn.ReLU)]},
                                                  ignore_layer=[ref.quantize.QuantMeasure], quant_op=False)
    graph, bottoms = tr.log.getGraph(), tr.log.getBottoms()
    names, nodes = {}, []
    for i, key in enumerate(graph):
        if key == "Data":
            nm, rec = "Data", dict(type="Data")
        elif isinstance(graph[key], str):
            nm, rec = key, dict(type="Func")
        else:
            nm = "m%d" % i
            rec = workload.describe_module(graph[key])
        names[key] = nm
        b = bottoms[key]
        rec.update(key=nm, bottoms=None if b is None else [names[x] for x in b])
        nodes.append(rec)
    topo = dict(name=name, input=list(data.shape), source="reference trace (PyTransformer), ReLU6 -> ReLU", nodes=nodes)
    with open(os.path.join(GOLD, "topology_%s.json" % name), "w") as f:
        json.dump(topo, f, separators=(",", ":"))
    print(name, len(nodes), "nodes")
    return topo


# ---------------------------------------------------------------------------------------------------------
def run_reference_pipeline(name, seed=0, signed=False, quantize=True, s_range=(1e-8, 1e8), delete_single=False):
    topo = workload.load_topology(os.path.join(GOLD, "topology_%s.json" % name))
    graph, bottoms, _ = workload.build_graph(topo, seed=seed)
    targ = [nn.Conv2d, nn.Linear]
    keys = list(graph.keys())
    pos = {k: i for i, k in enumerate(keys)}
    out = {}
    t0 = time.time()
    ref.layer_transform.merge_batchnorm(None, graph, bottoms, targ)
    rels = ref.relation.create_relation(graph, bottoms, targ, delete_single=delete_single)
    out["relations"] = np.array([[pos[a], pos[b], pos[c]] for a, b, c in (r.get_idxs() for r in rels)], np.int64)
    tl = [k for k in keys if type(graph[k]) in targ]
    out["targets"] = np.array([pos[k] for k in tl], np.int64)

    def stage(tag):
        dg = [digest(graph[k].weight) for k in tl]
        out[tag + "_w_sha"] = np.array([d[0] for d in dg])
        out[tag + "_w_absmax"] = np.array([d[1] for d in dg])
        out[tag + "_w_sum"] = np.array([d[2] for d in dg])
        for k in tl:
            if graph[k].bias is not None:
                out["%s_bias_%d" % (tag, pos[k])] = graph[k].bias.detach().numpy().copy()
        for k in keys:
            if hasattr(graph[k], "fake_bias") and not isinstance(graph[k], str):
                out["%s_fb_%d" % (tag, pos[k])] = graph[k].fake_bias.numpy().copy()
                out["%s_fw_%d" % (tag, pos[k])] = graph[k].fake_weight.numpy().copy()

    stage("fold")
    # count sweeps by wrapping _layer_equalization
    calls = [0]
    orig = ref.dfq._layer_equalization

    def counted(*a, **kw):
        calls[0] += 1
        return orig(*a, **kw)
    ref.dfq._layer_equalization = counted
    ref.dfq.cross_layer_equalization(graph, rels, targ, s_range=list(s_range), converge_thres=2e-7, signed=signed)
    ref.dfq._layer_equalization = orig
    out["n_sweeps"] = np.array(calls[0] // max(1, len(rels)))
    for i, r in enumerate(rels):
        out["S_%d" % i] = r.S.numpy().copy()
    stage("cle")
    ref.dfq.bias_correction(graph, bottoms, targ, signed=signed)
    stage("bc")
    if quantize:
        ref.layer_transform.quantize_targ_layer(graph, 8, 16, targ)
        stage("q")
    out["meta"] = np.array(json.dumps(dict(model=name, seed=seed, signed=signed, s_range=list(s_range),
                                           delete_single=delete_single, torch=torch.__version__,
                                           seconds=round(time.time() - t0, 1))))
    suffix = ("_signed" if signed else "")
    np.savez_compressed(os.path.join(GOLD, "ref_%s%s.npz" % (name, suffix)), **out)
    print(name, "sweeps", int(out["n_sweeps"]), "relations", len(rels), "%.1fs" % (time.time() - t0))


# ---------------------------------------------------------------------------------------------------------
def op_vectors():
    out = {}
    torch.manual_seed(1)
    shapes = {"dense_dw": ((32, 3, 3, 3), (32, 1, 3, 3)), "dw_pw": ((96, 1, 3, 3), (24, 96, 1, 1)),
              "pw_dw": ((144, 24, 1, 1), (144, 1, 3, 3)), "pw_pw": ((320, 96, 1, 1), (128, 320, 1, 1)),
              "pw_fc": ((128, 32, 1, 1), (10, 128)), "dense": ((64, 32, 3, 3), (48, 64, 3, 3)),
              "grouped": ((32, 8, 3, 3), (24, 16, 3, 3))}
    for tag, (s1, s2) in shapes.items():
        for signed in (False, True):
            w1 = torch.randn(*s1) * (10 ** torch.empty(s1[0]).uniform_(-1, 1)).view(-1, *([1] * (len(s1) - 1)))
            w2 = torch.randn(*s2)
            b1, bw, bb = torch.randn(s1[0]), torch.rand(s1[0]) + 0.5, torch.randn(s1[0])
            key = "eq_%s_%d" % (tag, int(signed))
            for n, t in (("w1", w1), ("w2", w2), ("b1", b1), ("bw", bw), ("bb", bb)):
                out["%s_in_%s" % (key, n)] = t.numpy().copy()
            r = ref.dfq._layer_equalization(w1, w2, b1, bw, bb, signed=signed)
            for n, t in (("w1", w1), ("w2", w2), ("b1", b1), ("bw", bw), ("bb", bb), ("S", r[3])):
                out["%s_out_%s" % (key, n)] = t.numpy().copy()
    # fake-quant codes on the reference's CPU path
    for bits in (8, 4, 16):
        for sym in (False, True):
            x = torch.randn(4096) * 3
            y = ref.quantize.quantize(x, bits, float(x.min()), float(x.max()), symmetric=sym)
            out["q_%d_%d_in" % (bits, int(sym))] = x.numpy().copy()
            out["q_%d_%d_out" % (bits, int(sym))] = y.numpy().copy()
    x = torch.randn(2000)
    out["qerr_in"] = x.numpy().copy()
    out["qerr_out"] = ref.dfq._quantize_error(x, 8, None).numpy().copy()
    out["qerr_out_signed"] = ref.dfq._quantize_error(x, 8, None, True).numpy().copy()
    # implicit-range path (bias quantization in Quant*/Q* layers, min_value=None)
    b = torch.randn(257)
    out["qimp_in"] = b.numpy().copy()
    out["qimp_out16"] = ref.quantize.quantize(b, num_bits=16).numpy().copy()
    out["qimp_out8"] = ref.quantize.quantize(b, num_bits=8).numpy().copy()
    # observer
    qm = ref.quantize.QuantMeasure(True)
    qm.eval()
    acts = torch.randn(8, 3, 16, 16)
    y = qm(acts)
    out["obs_in"] = acts.numpy().copy(); out["obs_out"] = y.numpy().copy()
    out["obs_min"] = np.array(float(qm.running_min)); out["obs_max"] = np.array(float(qm.running_max))
    qm2 = ref.quantize.QuantMeasure(False)
    qm2.train()
    y2 = qm2(acts)
    out["ema_out"] = y2.detach().numpy().copy()
    out["ema_min"] = np.array(float(qm2.running_min)); out["ema_max"] = np.array(float(qm2.running_max))
    # relu expectation as bias_correction forms it
    from scipy.stats import norm
    g = torch.rand(300) + 0.2; bta = torch.randn(300)
    e = g * torch.from_numpy(norm(0, 1).pdf(-bta / g)).float() + bta * (1 - torch.from_numpy(norm.cdf(-bta / g)).float())
    e[e < 0] = 0
    out["expect_g"] = g.numpy().copy(); out["expect_b"] = bta.numpy().copy(); out["expect_out"] = e.numpy().copy()
    np.savez_compressed(os.path.join(GOLD, "ref_ops.npz"), **out)
    print("ops", len(out))


if __name__ == "__main__":
    what = sys.argv[1:] or ["topology", "ops", "resnet18", "mobilenetv2"]
    os.makedirs(GOLD, exist_ok=True)
    if "topology" in what:
        for m in ("mobilenetv2", "resnet18", "deeplab", "ssd"):
            try:
                trace_topology(m)
            except Exception as e:  # noqa
                print("topology", m, "FAILED:", repr(e))
    if "ops" in what:
        op_vectors()
    if "resnet18" in what:
        run_reference_pipeline("resnet18", seed=3)
    if "mobilenetv2" in what:
        run_reference_pipeline("mobilenetv2", seed=0)
    if "mobilenetv2_signed" in what:
        run_reference_pipeline("mobilenetv2", seed=0, signed=True, quantize=False)
    if "deeplab" in what:
        run_reference_pipeline("deeplab", seed=5)
    if "ssd" in what:
        run_reference_pipeline("ssd", seed=7, delete_single=True)


# ---------------------------------------------------------------------------------------------------------
def quant_minmax_fixture(name="mobilenetv2", seed=0):
    """set_quant_minmax (layer_transform.py:347-609) needs the tracer's record of functional ops; trace the reference
    model with Quant layers + observers, store the op record with the topology, run the reference calibration on the
    seeded topology-built graph and store every observer's running_min / running_max."""
    TT = refenv.tracer()
    Q = ref.quantize
    if name == "mobilenetv2":
        from modeling.classification.MobileNetV2 import mobilenet_v2
        model, data = mobilenet_v2(None), torch.ones((4, 3, 224, 224))
    elif name == "resnet18":
        import torchvision.models as models
        model, data = models.resnet18(), torch.ones((4, 3, 224, 224))
    model.eval()
    tr = TT()
    md = {0: [(nn.ReLU6, nn.ReLU)], 1: [(nn.Conv2d, Q.QuantNConv2d), (nn.Linear, Q.QuantNLinear)]}
    model, tr = ref.layer_transform.switch_layers(model, tr, data, md, ignore_layer=[Q.QuantMeasure], quant_op=True)
    record = [list(x) for x in model.name_tensor_op]
    topo = workload.load_topology(os.path.join(GOLD, "topology_%s.json" % name))
    graph0 = tr.log.getGraph()
    assert len(graph0) == len(topo["nodes"]), (len(graph0), len(topo["nodes"]))
    topo["tensor_ops"] = record
    with open(os.path.join(GOLD, "topology_%s.json" % name), "w") as f:
        json.dump(topo, f, separators=(",", ":"))
    # reference calibration on the seeded graph built from the topology, with the reference's own Quant classes
    graph, bottoms, _ = workload.build_graph(topo, seed=seed, conv_cls=Q.QuantNConv2d, linear_cls=Q.QuantNLinear)
    targ = [Q.QuantNConv2d, Q.QuantNLinear]
    LT = ref.layer_transform
    ops = []
    for _, op_name in record:
        ops.extend(Q.QuantMeasure(num_bits=8, momentum=0.1) for _ in range(int(op_name.split('_')[-1])))
    LT.module_tensor_op = LT.CustomTensorOP(ops, [tuple(x) for x in record])
    LT.merge_batchnorm(None, graph, bottoms, targ)
    rels = ref.relation.create_relation(graph, bottoms, targ)
    ref.dfq.cross_layer_equalization(graph, rels, targ, converge_thres=2e-7)
    ref.dfq.bias_correction(graph, bottoms, targ)
    LT.set_quant_minmax(graph, bottoms, verbose=False)
    out = {}
    for i, k in enumerate(graph):
        m = graph[k]
        if hasattr(m, "quant") and not isinstance(m, str):
            out["layer_%d" % i] = np.array([float(m.quant.running_min), float(m.quant.running_max)])
    for j, qm in enumerate(ops):
        out["op_%d" % j] = np.array([float(qm.running_min), float(qm.running_max)])
    np.savez_compressed(os.path.join(GOLD, "ref_minmax_%s.npz" % name), **out)
    print("minmax", name, len(out), "observers;", len(record), "functional ops")


if __name__ == "__main__" and "minmax" in sys.argv[1:]:
    quant_minmax_fixture("mobilenetv2", 0)
    quant_minmax_fixture("resnet18", 3)


# ---------------------------------------------------------------------------------------------------------
def bias_correction_fixture(name):
    """dfq.py:173-293 alone: inputs from tests/bc_fixture.py, outputs of the reference."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import bc_fixture
    graph, bottoms = bc_fixture.build(name)
    out = {"digests": bc_fixture.input_digests(graph), "seed": np.array(bc_fixture.SEEDS[name])}
    ref.dfq.bias_correction(graph, bottoms, bc_fixture.TARG)
    n = 0
    for i, k in enumerate(graph):
        m = graph[k]
        if type(m) in bc_fixture.TARG and m.bias is not None:
            out["out_b_%d" % i] = m.bias.detach().numpy().copy(); n += 1
        elif hasattr(m, "fake_bias") and not isinstance(m, str):
            out["out_fb_%d" % i] = m.fake_bias.numpy().copy()
    np.savez_compressed(os.path.join(GOLD, "ref_bc_%s.npz" % name), **out)
    print("bc", name, n, "corrected layers")


if __name__ == "__main__" and "bc" in sys.argv[1:]:
    bias_correction_fixture("resnet18")
    bias_correction_fixture("mobilenetv2")


# ---------------------------------------------------------------------------------------------------------
def ncnn_table_rows():
    """The 53 + 53 scale values of the reference's checked-in table (modeling/ncnn/model_quant_relu_equal.table): rows 1-53
    `<layer>_param_0 s s s ...` (first value = 128/max|W|), rows 54-106 `<layer> s` (activation scale)."""
    rows = [l.split() for l in open(os.path.join(refenv.REF_ROOT, "modeling", "ncnn", "model_quant_relu_equal.table")).read().strip().splitlines()]
    assert len(rows) == 106
    np.savez_compressed(os.path.join(GOLD, "ncnn_table_rows.npz"), weight_scales=np.array([float(r[1]) for r in rows[:53]]),
                        activation_scales=np.array([float(r[1]) for r in rows[53:]]),
                        names=np.array([r[0] for r in rows[53:]]))
    print("ncnn table rows: 53 + 53")


if __name__ == "__main__" and "table" in sys.argv[1:]:
    ncnn_table_rows()


# ---------------------------------------------------------------------------------------------------------
def live_pins():
    """What the pin tests used to compute by importing the reference at test time, stored so that they run anywhere:
    _layer_equalization on the CASES of tests/test_oracle_pins.py (sha256 of every output tensor), the replace_op forward of
    tests/test_op_patching.py (outputs and observer order) and getDistilData on tests/test_distill.py's tiny model (a seeded
    sample of 4096 pixels per batch plus each batch's fp64 sum)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_oracle_pins as P
    out = {}
    for ci, (s1, s2, opt) in enumerate(P.CASES):
        for signed in (False, True):
            torch.manual_seed(hash((s1, s2, signed)) % 1000)
            opt_ = dict(opt)
            degenerate = opt_.pop("degenerate", False)
            w1 = torch.randn(*s1) * (10 ** torch.empty(s1[0]).uniform_(-1, 1)).view(-1, *([1] * (len(s1) - 1)))
            w2 = torch.randn(*s2)
            if degenerate:
                w1[1] = 0; w1[3] = 0.5
                w2.view(s2[0], s2[1], -1)[:, 2] = 0
            b1, bw, bb = torch.randn(s1[0]), torch.rand(s1[0]) + 0.5, torch.randn(s1[0])
            key = "eq_%d_%d" % (ci, int(signed))
            out[key + "_in"] = np.array([P.sha256(t.numpy()) for t in (w1, w2, b1, bw, bb)])
            r = ref.dfq._layer_equalization(w1, w2, b1, bw, bb, signed=signed, **opt_)
            out[key + "_out"] = np.array([P.sha256(t.numpy()) for t in (w1, w2, b1, bw, bb, r[3])])

    import test_op_patching as T
    torch.manual_seed(0)
    model = T.Net().eval()
    x = torch.randn(2, 3, 6, 6)
    theirs, seen, _ = T._run_patched(ref.layer_transform, ref.quantize.QuantMeasure, model, x)
    out["patch_seen"] = np.array([i for i, _ in seen])
    for k, t in enumerate(theirs):
        out["patch_out_%d" % k] = t.numpy()

    import run_main
    import test_distill as D
    run_main.prepare_environment(use_dropin=False)
    from ZeroQ.distill_data import getDistilData as ref_get
    model = D._tiny()
    torch.manual_seed(123)
    theirs = ref_get(model, "imagenet", 2, num_batch=2, gpu=False, value_range=[-2.11790393, 2.64], early_break_factor=1e9)
    for k, t in enumerate(theirs):
        a = t.detach().numpy()
        out["distill_shape_%d" % k] = np.array(a.shape)
        out["distill_sum_%d" % k] = np.array(a.astype(np.float64).sum())
        out["distill_sample_%d" % k] = a.reshape(-1)[D.sample_index(a.size)]
    np.savez_compressed(os.path.join(GOLD, "ref_live_pins.npz"), **out)
    print("live pins:", len(out), "arrays")


if __name__ == "__main__" and "live" in sys.argv[1:]:
    live_pins()


# ---------------------------------------------------------------------------------------------------------
SSD_POST_CONFIGS = [(-1, 200), (1, 200), (5, 200), (-1, 1)]     # (top_k, candidate_size)


def ssd_postprocess():
    """The reference's Predictor.predict post-processing (box_utils decode, threshold, sort, hard_nms, scaling) run on
    seeded SSD-Lite-shaped outputs with the priors of mobilenetv1_ssd_config (3,000 x 4), for each (top_k, candidate_size)
    of SSD_POST_CONFIGS.  Image 0 has a class without candidates, image 2 no detection at all; no class has tied scores,
    so the unstable sort does not decide anything."""
    from modeling.detection.config import mobilenetv1_ssd_config as cfg
    from modeling.detection.predictor import Predictor
    priors = cfg.priors.float().contiguous()
    P, C = priors.shape[0], 21
    g = torch.Generator().manual_seed(7)
    logits = torch.randn(3, P, C, generator=g) * 2.5
    logits[..., 0] += 5.0
    logits[0, :, 5] -= 30.0                       # no candidate of class 5 in image 0
    logits[1, :, 1:] *= 1.6                       # a peakier image
    logits[2, :, 0] += 40.0                       # nothing above the threshold
    scores = torch.softmax(logits, dim=2)
    locations = torch.randn(3, P, 4, generator=g) * 0.7
    sizes = np.array([[300, 300], [640, 480], [333, 500]], np.int64)
    for n in range(3):
        for c in range(1, C):
            s = scores[n, :, c]
            assert torch.unique(s[s > 0.01]).numel() == int((s > 0.01).sum()), "tied scores"

    class Outputs(nn.Module):
        def forward(self, x):
            return self.scores, (self.locations, priors, cfg.center_variance, cfg.size_variance)

    net = Outputs()
    out = dict(scores=scores.numpy(), locations=locations.numpy(), priors=priors.numpy(), image_sizes=sizes,
               variances=np.array([cfg.center_variance, cfg.size_variance]), prob_threshold=np.array(0.01),
               iou_threshold=np.array(cfg.iou_threshold), configs=np.array(SSD_POST_CONFIGS))
    for k, (top_k, cand) in enumerate(SSD_POST_CONFIGS):
        pred = Predictor(net, cfg.image_size, cfg.image_mean, cfg.image_std, iou_threshold=cfg.iou_threshold,
                         candidate_size=cand, device=torch.device("cpu"))
        boxes, labels, probs, offs = [], [], [], [0]
        for n in range(3):
            net.scores, net.locations = scores[n:n + 1], locations[n:n + 1]
            w, h = (int(v) for v in sizes[n])
            b, l, p = pred.predict(np.zeros((h, w, 3), np.uint8), top_k=top_k, prob_threshold=0.01)
            boxes.append(b.reshape(-1, 4)); labels.append(l.reshape(-1).long()); probs.append(p.reshape(-1))
            offs.append(offs[-1] + b.shape[0])
        out["boxes_%d" % k] = torch.cat(boxes).numpy()
        out["labels_%d" % k] = torch.cat(labels).numpy()
        out["probs_%d" % k] = torch.cat(probs).numpy()
        out["offsets_%d" % k] = np.array(offs)
        print("ssd postprocess top_k %d candidate_size %d: kept per image %s" % (top_k, cand, np.diff(offs).tolist()))
    np.savez_compressed(os.path.join(GOLD, "ref_ssd_postprocess.npz"), **out)


if __name__ == "__main__" and "ssd_post" in sys.argv[1:]:
    ssd_postprocess()


SSD_SOFT_TOP_K = [-1, 1, 5]
SSD_SOFT_SIGMA = 0.3


def ssd_soft_nms():
    """The reference's Predictor(nms_method="soft", sigma=SSD_SOFT_SIGMA).predict (box_utils decode, threshold,
    soft_nms, scaling) on the CPU, run on two seeded SSD-Lite-shaped images with the priors of mobilenetv1_ssd_config
    (3,000 x 4), for each top_k of SSD_SOFT_TOP_K.  Image 1 is peakier and has a class without candidates."""
    from modeling.detection.config import mobilenetv1_ssd_config as cfg
    from modeling.detection.predictor import Predictor
    priors = cfg.priors.float().contiguous()
    P, C = priors.shape[0], 21
    g = torch.Generator().manual_seed(11)
    logits = torch.randn(2, P, C, generator=g) * 2.5
    logits[..., 0] += 5.0
    logits[1, :, 1:] *= 1.6
    logits[1, :, 7] -= 40.0                       # no candidate of class 7 in image 1
    scores = torch.softmax(logits, dim=2)
    locations = torch.randn(2, P, 4, generator=g) * 0.7
    sizes = np.array([[500, 375], [300, 300]], np.int64)

    class Outputs(nn.Module):
        def forward(self, x):
            return self.scores, (self.locations, priors, cfg.center_variance, cfg.size_variance)

    net = Outputs()
    out = dict(scores=scores.numpy(), locations=locations.numpy(), priors=priors.numpy(), image_sizes=sizes,
               variances=np.array([cfg.center_variance, cfg.size_variance]), prob_threshold=np.array(0.01),
               sigma=np.array(SSD_SOFT_SIGMA), top_ks=np.array(SSD_SOFT_TOP_K))
    pred = Predictor(net, cfg.image_size, cfg.image_mean, cfg.image_std, nms_method="soft", sigma=SSD_SOFT_SIGMA,
                     device=torch.device("cpu"))
    for k, top_k in enumerate(SSD_SOFT_TOP_K):
        boxes, labels, probs, offs = [], [], [], [0]
        for n in range(2):
            net.scores, net.locations = scores[n:n + 1], locations[n:n + 1]
            w, h = (int(v) for v in sizes[n])
            b, l, p = pred.predict(np.zeros((h, w, 3), np.uint8), top_k=top_k, prob_threshold=0.01)
            boxes.append(b.reshape(-1, 4)); labels.append(l.reshape(-1).long()); probs.append(p.reshape(-1))
            offs.append(offs[-1] + b.shape[0])
        out["boxes_%d" % k] = torch.cat(boxes).numpy()
        out["labels_%d" % k] = torch.cat(labels).numpy()
        out["probs_%d" % k] = torch.cat(probs).numpy()
        out["offsets_%d" % k] = np.array(offs)
        print("ssd soft nms top_k %d: kept per image %s" % (top_k, np.diff(offs).tolist()))
    np.savez_compressed(os.path.join(GOLD, "ref_ssd_soft_nms.npz"), **out)


if __name__ == "__main__" and "ssd_soft" in sys.argv[1:]:
    ssd_soft_nms()


# ---------------------------------------------------------------------------------------------------------
def seg_eval():
    """forward_all's per-batch steps (utils/segmentation/utils.py) on three seeded batches of full-resolution logits
    [2, 21, 20, 28] and float32 labels, as the reference's dataset yields them: torch.max(logits, 1)[1] as uint8, the
    labels through astype(np.uint8), then the reference's own Evaluator.add_batch.  Batch 0 has logits rounded to a coarse
    grid (many tied maxima) and labels with 255 borders and fractional values (-0.5 .. 20.9); batch 1 has no pixel of class
    7 in its labels; batch 2 is all 255.  Stores the matrix after each add_batch and the four metrics of each, and those of
    a fresh Evaluator given the all-255 batch alone (an empty matrix: NaN metrics)."""
    from utils.metrics import Evaluator
    g = torch.Generator().manual_seed(5)
    N, C, H, W = 2, 21, 20, 28
    out = {}
    ev = Evaluator(C)

    def metrics(e):
        with np.errstate(all="ignore"):
            return np.array([e.Pixel_Accuracy(), e.Pixel_Accuracy_Class(), e.Mean_Intersection_over_Union(),
                             e.Frequency_Weighted_Intersection_over_Union()])
    for b in range(3):
        logits = torch.randn(N, C, H, W, generator=g)
        logits[:, 0] += 0.8                                       # background most likely, as in VOC
        if b == 0:
            logits = torch.round(logits * 2) / 2
        labels = torch.randint(0, C, (N, H, W), generator=g).float()
        labels[torch.rand(N, H, W, generator=g) < 0.5] = 0.
        if b == 0:
            labels += torch.rand(N, H, W, generator=g).mul(0.9)    # fractional values truncate toward zero
            labels[0, 5, :5] = -0.5
        if b == 1:
            labels[labels == 7] = 3.
        labels[:, :2] = 255.
        labels[:, :, -1] = 255.
        if b == 2:
            labels[:] = 255.
        pred = torch.max(logits, 1)[1].numpy().astype(np.uint8)
        lab = labels.numpy().astype(np.uint8)
        ev.add_batch(lab, pred)
        out.update({"logits_%d" % b: logits.numpy(), "labels_%d" % b: labels.numpy(), "pred_%d" % b: pred,
                    "matrix_%d" % b: ev.confusion_matrix.copy(), "metrics_%d" % b: metrics(ev)})
        print("seg eval batch %d: %d pixels counted, metrics %s" % (b, int(ev.confusion_matrix.sum()), metrics(ev)))
    empty = Evaluator(C)
    empty.add_batch(out["labels_2"].astype(np.uint8), out["pred_2"])
    out["matrix_empty"], out["metrics_empty"] = empty.confusion_matrix.copy(), metrics(empty)
    np.savez_compressed(os.path.join(GOLD, "ref_seg_eval.npz"), **out)


if __name__ == "__main__" and "seg_eval" in sys.argv[1:]:
    seg_eval()


# ---------------------------------------------------------------------------------------------------------
SSD_MAP_CONFIGS = [(0.5, True), (0.5, False), (0.55, True), (0.55, False)]     # (iou_threshold, use_2007_metric)


def _ulp_search(x0, f, want, n=20000):
    """The fp32 x nearest to x0, within n ulps either side, with want(f(x)) true."""
    k = np.arange(-n, n, dtype=np.float32)
    k = k[np.argsort(np.abs(k), kind="stable")]
    xs = torch.from_numpy(np.float32(x0) + k * np.spacing(np.float32(x0)))
    hit = torch.nonzero(want(f(xs))).reshape(-1)
    assert hit.numel(), "no seeded box found"
    return np.float32(xs[hit[0]])


def ssd_map_scene():
    """Seeded detections and annotations for 9 classes (class 8 has no ground truth) in which each rule of DESIGN.md
    section 3.11 decides an AP: a random scene of jittered copies of the annotations plus clutter, and constructed images
    for the +1/-1 rounding, an IoU equal to float32(0.55), a second detection on one box, a difficult argmax next to a
    passing non-difficult box, equal IoUs, a class whose best detection hits a difficult box, detections on images
    without boxes of their class, a class without detections (6) and NaN boxes.  No class has tied scores."""
    g = np.random.default_rng(11)
    C = 9
    gts, dets = [], []

    def add(gt, det):                     # gt [(box, label, difficult)], det [(box, label, score)]
        gts.append((np.array([b for b, _, _ in gt], np.float32).reshape(-1, 4) if gt else np.array([], np.float32),
                    np.array([l for _, l, _ in gt], np.int64), np.array([d for _, _, d in gt], np.uint8)))
        dets.append(det)
    # random scene: 24 images, classes 1 .. 5 and 7
    for n in range(24):
        gt, det = [], []
        for _ in range(int(g.integers(0, 6))):
            x1, y1 = g.uniform(0, 400, 2)
            w, h = g.uniform(20, 200, 2)
            gt.append(([x1, y1, min(x1 + w, 500), min(y1 + h, 500)], int(g.choice([1, 2, 3, 4, 5, 7])),
                       int(g.random() < 0.2)))
        for b, l, _ in gt:
            for _ in range(int(g.integers(0, 4))):
                det.append((np.float32(np.array(b) + g.normal(0, 12, 4)), l, None))
        for _ in range(int(g.integers(0, 6))):
            x1, y1 = g.uniform(0, 400, 2)
            det.append((np.float32([x1, y1, x1 + g.uniform(10, 100), y1 + g.uniform(10, 100)]),
                        int(g.choice([1, 2, 3, 4, 5, 7])), None))
        add(gt, det)
    # the +1/-1 rounding moves an IoU across the threshold: box x2 in [255, 256), where b + 1 loses a bit
    for thr in (0.5, 0.55):
        gx1 = np.float32(255.0 - thr * 400.0)
        for y2 in range(300, 400):                   # the first box height with a crossing near x2 = 255
            gt = [gx1, 40.0, gx1 + 400.0, float(y2)]

            def iou_x2(xs, plus_one):
                b = torch.stack([torch.full_like(xs, gx1), torch.full_like(xs, 40.0), xs, torch.full_like(xs, float(y2))], 1)
                if plus_one:
                    b = (b + 1.0) - 1.0
                return _ref_iou_of(b, torch.tensor([gt], dtype=torch.float32))
            try:
                x2 = _ulp_search(255.0, lambda xs: torch.stack([iou_x2(xs, False), iou_x2(xs, True)]),
                                 lambda v: (v[0].double() > thr) != (v[1].double() > thr))
                break
            except AssertionError:
                continue
        add([(gt, 1, 0)], [(np.float32([gx1, 40.0, x2, y2]), 1, None)])
    # an fp32 IoU equal to float32(0.55): above 0.55 in float64, not in fp32
    gt = [55.0, 40.0, 455.0, 300.0]

    def iou_55(xs):
        b = torch.stack([torch.full_like(xs, 55.0), torch.full_like(xs, 40.0), xs, torch.full_like(xs, 300.0)], 1)
        return _ref_iou_of((b + 1.0) - 1.0, torch.tensor([gt], dtype=torch.float32))
    x2 = _ulp_search(274.99, iou_55, lambda v: v == np.float32(0.55))
    add([(gt, 2, 0)], [(np.float32([55.0, 40.0, x2, 300.0]), 2, None)])
    # two detections on one box: the second is a false positive
    add([([100., 100., 200., 200.], 1, 0)], [(np.float32([101, 100, 200, 201]), 1, None),
                                            (np.float32([100, 99, 199, 200]), 1, None)])
    # the argmax is a difficult box while a non-difficult one also passes: ignored
    add([([50., 50., 150., 150.], 2, 1), ([56., 52., 150., 152.], 2, 0)], [(np.float32([50, 50, 150, 150]), 2, None)])
    # equal IoU against two boxes (difficult first): the first wins, so the detection is ignored
    add([([90., 100., 190., 200.], 3, 1), ([110., 100., 210., 200.], 3, 0)], [(np.float32([100, 100, 200, 200]), 3, None)])
    # class 4's best detection hits a difficult box: NaN under the 2007 metric, finite under the area metric
    add([([300., 300., 400., 420.], 4, 1), ([20., 30., 120., 90.], 4, 0)],
        [(np.float32([300, 300, 400, 420]), 4, 0.9999), (np.float32([20, 30, 120, 90]), 4, 0.9998)])
    # detections of class 5 on images without boxes of class 5 (one without any box)
    add([([10., 10., 60., 60.], 1, 0)], [(np.float32([10, 10, 60, 60]), 5, 0.9997)])
    add([], [(np.float32([200, 200, 260, 280]), 5, 0.9996), (np.float32([5, 5, 50, 50]), 7, None)])
    # class 6 has boxes but no detection
    add([([30., 40., 230., 240.], 6, 0), ([40., 40., 90., 90.], 6, 1)], [])
    # NaN boxes: a ground-truth box with a NaN first (every IoU against it NaN wins), and a NaN detection
    add([([np.nan, 300., 400., 400.], 7, 0), ([10., 10., 110., 110.], 7, 0)], [(np.float32([10, 10, 110, 110]), 7, 0.9995)])
    add([([10., 10., 110., 110.], 7, 0)], [(np.float32([10, np.nan, 110, 110]), 7, 0.9994)])
    # class 8 has detections but no ground truth: the reference raises KeyError
    add([], [(np.float32([0, 0, 30, 30]), 8, 0.5)])
    # scores: the given ones, the rest random, unique within each class
    out = []
    for det in dets:
        rows = [(b, l, np.float32(s) if s is not None else np.float32(g.uniform(0.011, 0.99))) for b, l, s in det]
        rows.sort(key=lambda r: (r[1], -r[2]))            # classes ascending, score descending, as postprocess returns
        out.append((torch.tensor(np.array([r[0] for r in rows], np.float32).reshape(-1, 4)),
                    torch.tensor([r[1] for r in rows], dtype=torch.int64), torch.tensor([r[2] for r in rows])))
    for c in range(1, C):
        s = torch.cat([p[l == c] for _, l, p in out])
        assert torch.unique(s).numel() == s.numel(), "tied scores in class %d" % c
    return C, gts, out


def _ref_iou_of(boxes, gt):
    """box_utils.iou_of(boxes, gt) for the searches above (the reference's own function)."""
    from utils.detection import box_utils
    return box_utils.iou_of(boxes, gt)


def ssd_map():
    """main_ssd.py's evaluation on ssd_map_scene(): the per-class files written exactly as the main's loop writes them,
    group_annotation_by_class on a stand-in dataset and compute_average_precision_per_class per class, for each
    (iou_threshold, use_2007_metric) of SSD_MAP_CONFIGS.  A KeyError (class 8) is stored as NaN."""
    import tempfile
    saved = sys.argv
    sys.argv = ["main_ssd.py"]
    import main_ssd
    sys.argv = saved
    C, gts, dets = ssd_map_scene()

    class Dataset:
        ids = ["%06d" % n for n in range(len(gts))]

        def __len__(self):
            return len(self.ids)

        def get_annotation(self, i):
            return self.ids[i], gts[i]
    dataset = Dataset()
    true_case_stat, all_gb_boxes, all_difficult_cases = main_ssd.group_annotation_by_class(dataset)
    results = []
    for i, (boxes, labels, probs) in enumerate(dets):
        indexes = torch.ones(labels.size(0), 1, dtype=torch.float32) * i
        results.append(torch.cat([indexes.reshape(-1, 1), labels.reshape(-1, 1).float(), probs.reshape(-1, 1),
                                  boxes + 1.0], dim=1))
    results = torch.cat(results)
    out = dict(num_classes=np.array(C), configs=np.array(SSD_MAP_CONFIGS, np.float64))
    with tempfile.TemporaryDirectory() as tmp:
        for c in range(1, C):
            with open(os.path.join(tmp, "det_test_%d.txt" % c), "w") as f:
                sub = results[results[:, 1] == c, :]
                for i in range(sub.size(0)):
                    prob_box = sub[i, 2:].numpy()
                    print(dataset.ids[int(sub[i, 0])] + " " + " ".join([str(v) for v in prob_box]), file=f)
        for k, (thr, use_2007) in enumerate(SSD_MAP_CONFIGS):
            aps = []
            for c in range(1, C):
                try:
                    with np.errstate(all="ignore"):
                        aps.append(main_ssd.compute_average_precision_per_class(
                            true_case_stat[c], all_gb_boxes[c], all_difficult_cases[c],
                            os.path.join(tmp, "det_test_%d.txt" % c), thr, use_2007))
                except KeyError:
                    aps.append(np.nan)
            out["aps_%d" % k] = np.array(aps, np.float64)
            print("ssd map iou %.2f 2007 %s: %s" % (thr, use_2007, out["aps_%d" % k]))
    out["gt_boxes"] = np.concatenate([b.reshape(-1, 4) for b, _, _ in gts])
    out["gt_labels"] = np.concatenate([l for _, l, _ in gts])
    out["gt_difficult"] = np.concatenate([d for _, _, d in gts])
    out["gt_offsets"] = np.cumsum([0] + [len(l) for _, l, _ in gts])
    out["det_boxes"] = torch.cat([b for b, _, _ in dets]).numpy()
    out["det_labels"] = torch.cat([l for _, l, _ in dets]).numpy()
    out["det_probs"] = torch.cat([p for _, _, p in dets]).numpy()
    out["det_offsets"] = np.cumsum([0] + [l.numel() for _, l, _ in dets])
    np.savez_compressed(os.path.join(GOLD, "ref_ssd_map.npz"), **out)


if __name__ == "__main__" and "ssd_map" in sys.argv[1:]:
    ssd_map()


# ---------------------------------------------------------------------------------------------------------
def preprocess():
    """The reference's evaluation transforms on the seeded images of tests/preprocess_cases.py: torchvision's
    Resize(256) / CenterCrop(224) / ToTensor / Normalize (main_cls.py), VOCSegmentation.transform_val's FixScaleCrop(513) /
    Normalize / ToTensor (custom_transforms), and PredictionTransform(300, 127, 128) (main_ssd.py).  Stores the sha256 of
    each float32 output's bytes: the tests compare bit for bit, and the outputs themselves are megabytes each."""
    import hashlib
    from PIL import Image
    from torchvision import transforms
    import dataset.segmentation.custom_transforms as tr
    from modeling.detection.data_preprocessing import PredictionTransform
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import preprocess_cases as PC
    cls = transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224), transforms.ToTensor(),
                              transforms.Normalize((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))])
    seg = transforms.Compose([tr.FixScaleCrop(crop_size=513), tr.Normalize(mean=(0.485, 0.456, 0.406),
                                                                              std=(0.229, 0.224, 0.225)), tr.ToTensor()])
    ssd = PredictionTransform(300, np.array([127, 127, 127]), 128.0)

    def sha(t):
        return hashlib.sha256(np.ascontiguousarray(t.numpy(), np.float32).tobytes()).hexdigest()
    out = {"names": np.array([c[0] for c in PC.cases()])}
    for name, img, lab in PC.cases():
        h, w = img.shape[:2]
        c = cls(Image.fromarray(img))
        out["cls_" + name] = sha(c)
        s = seg({"image": Image.fromarray(img), "label": Image.fromarray(lab)})
        out["seg_" + name], out["seglab_" + name] = sha(s["image"]), sha(s["label"])
        d = ssd(img)
        out["ssd_" + name] = sha(d)
        print("preprocess %s: cls %s seg %s ssd %s" % (name, out["cls_" + name][:8], out["seg_" + name][:8],
                                                     out["ssd_" + name][:8]))
    np.savez_compressed(os.path.join(GOLD, "ref_preprocess.npz"), **out)


if __name__ == "__main__" and "preprocess" in sys.argv[1:]:
    preprocess()


# ---------------------------------------------------------------------------------------------------------
def absorb_clip_fixture():
    """dfq.py:121-170 between the equalization and the correction, in the mains' order, on tests/absorb_clip_case.py."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import absorb_clip_case as case
    targ = [nn.Conv2d, nn.Linear]
    out = {}
    for name, seed, n, clip in case.FIXTURE_CASES:
        graph, bottoms, _ = workload.build_graph(case.topology(name), seed=seed)
        keys = list(graph.keys())
        pos = {k: i for i, k in enumerate(keys)}

        def stage(tag):
            for k in keys:
                m = graph[k]
                if type(m) in targ:
                    if tag in ("cle", "clip"):      # absorption and correction leave the weights alone
                        out["%s_%s_w_%d" % (name, tag, pos[k])] = m.weight.detach().numpy().copy()
                    if m.bias is not None:
                        out["%s_%s_b_%d" % (name, tag, pos[k])] = m.bias.detach().numpy().copy()
                elif hasattr(m, "fake_bias") and not isinstance(m, str):
                    out["%s_%s_fw_%d" % (name, tag, pos[k])] = m.fake_weight.numpy().copy()
                    out["%s_%s_fb_%d" % (name, tag, pos[k])] = m.fake_bias.numpy().copy()
        ref.layer_transform.merge_batchnorm(None, graph, bottoms, targ)
        rels = ref.relation.create_relation(graph, bottoms, targ)
        out[name + "_relations"] = np.array([[pos[a], pos[b], pos[c]] for a, b, c in (r.get_idxs() for r in rels)], np.int64)
        ref.dfq.cross_layer_equalization(graph, rels, targ)
        stage("cle")
        ref.dfq.bias_absorption(graph, rels, bottoms, n)
        stage("absorb")
        ref.dfq.clip_weight(graph, list(clip), targ)
        stage("clip")
        ref.dfq.bias_correction(graph, bottoms, targ)
        stage("bc")
        out[name + "_meta"] = np.array(json.dumps(dict(seed=seed, N=n, clip=list(clip), torch=torch.__version__)))
    np.savez_compressed(os.path.join(GOLD, "ref_absorb_clip.npz"), **out)
    print("absorb_clip", len(out), "arrays")


if __name__ == "__main__" and "absorb_clip" in sys.argv[1:]:
    absorb_clip_fixture()
