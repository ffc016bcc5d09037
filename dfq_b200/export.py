"""On-disk outputs adjacent to the calibration path (SURVEY.md section 8f, rank 4).

  write_ncnn_table   the int8 calibration table the reference produces in convert_ncnn.py:178-201: one row per target
                     layer with the weight scale 128/max|W| repeated per output channel (`<name>_param_0 s s s ...`),
                     then one row per layer with the activation scale 128/max(|running_min|, |running_max|) (`<name> s`).
                     The per-tensor extrema are computed on the device (dfq_minmax).
  read_ncnn_table    the inverse of write_ncnn_table: (names, rows) in ncnn_scales' format, so a table - the reference's own
                     included - can drive int8.convert_to_int8.
  save_calibration   equalized / corrected state (weights, biases, fake BN statistics, scale vectors) as one .pt file.
"""
import torch

from .utils.quantize import tensor_minmax


def _scale128(extent, zero_ok):
    """128 / extent; a zero extent (all-zero weights, an activation range of 0) gives 0 when zero_ok, else raises."""
    return 0.0 if (zero_ok and extent == 0) else 128. / extent


def ncnn_scales(graph, targ_type, zero_range_ok=False):
    """[(weight_scale, out_channels, activation_scale | None)] per target layer, in graph order.  zero_range_ok: a zero
    range gives scale 0 (codes 0) instead of raising ZeroDivisionError."""
    rows = []
    for key in graph:
        layer = graph[key]
        if type(layer) not in targ_type:
            continue
        mm = tensor_minmax(layer.weight.detach()).tolist()                     # convert_ncnn.py:186-187
        w_scale = _scale128(max(abs(mm[1]), abs(mm[0])), zero_range_ok)
        a_scale = None
        if hasattr(layer, "quant"):
            mi, ma = float(torch.min(layer.quant.running_min)), float(torch.max(layer.quant.running_max))
            a_scale = _scale128(max(abs(ma), abs(mi)), zero_range_ok)         # :189-191
        rows.append((w_scale, layer.weight.shape[0], a_scale))
    return rows


def write_ncnn_table(graph, path, targ_type, names=None):
    """Write the table; `names` are the ncnn blob names of the target layers (default: layer_<i>)."""
    rows = ncnn_scales(graph, targ_type)
    names = names or ["layer_%d" % i for i in range(len(rows))]
    with open(path, "w") as f:
        for n, (ws, oc, _) in zip(names, rows):
            f.write(' '.join(["%s_param_0" % n] + [str(ws)] * oc) + '\n')
        for n, (_, _, a) in zip(names, rows):
            if a is not None:
                f.write("%s %s\n" % (n, str(a)))
    return rows


def read_ncnn_table(path):
    """(names, rows) of a table write_ncnn_table (or convert_ncnn.py) wrote: rows[i] = (weight_scale, out_channels,
    activation_scale | None), as ncnn_scales returns them.  A weight row whose values differ raises ValueError: the
    scheme has one weight scale per layer."""
    names, wrows, acts = [], [], {}
    with open(path) as f:
        for line in f:
            parts = line.split()
            if not parts:
                continue
            if parts[0].endswith("_param_0"):
                vals = [float(v) for v in parts[1:]]
                if any(v != vals[0] for v in vals):
                    raise ValueError("%s: per-channel weight scales of %s differ" % (path, parts[0]))
                names.append(parts[0][:-len("_param_0")])
                wrows.append((vals[0], len(vals)))
            else:
                acts[parts[0]] = float(parts[1])
    return names, [(ws, oc, acts.get(n)) for n, (ws, oc) in zip(names, wrows)]


def save_calibration(graph, relations, path):
    """Persist what the passes changed: parameters of every module with weights, fake BN statistics and Relation.S."""
    state = {"layers": {}, "bn": {}, "S": [None if r.S is None else r.S.detach().cpu() for r in relations]}
    for i, key in enumerate(graph):
        m = graph[key]
        if isinstance(m, str):
            continue
        if hasattr(m, "fake_weight"):
            state["bn"][i] = {"fake_weight": m.fake_weight.detach().cpu(), "fake_bias": m.fake_bias.detach().cpu()}
        elif hasattr(m, "weight") and m.weight is not None:
            state["layers"][i] = {"weight": m.weight.detach().cpu(), "bias": None if m.bias is None else m.bias.detach().cpu()}
    torch.save(state, path)
    return state
