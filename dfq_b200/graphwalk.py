"""Pure-Python graph walks of the calibration path (no tensor arithmetic).

`graph` / `bottoms` are the OrderedDicts the reference's tracer produces (SURVEY.md section 8b):
``graph[key]`` is an nn.Module or, for functional ops, the key string itself ("add_63", "torch.cat_7",
"torch.mean_150", ...); ``bottoms[key]`` lists the keys feeding it (None for the root).

  find_prev_bn             utils/layer_transform.py:299-344
  bias_correction_recipe   the control flow of dfq.py:186-293 with the tensor work factored out:
                           which BNs (rectified or not) make up E[x] of each corrected layer, how they are
                           merged (cat / add), and which BN's fake_bias receives -delta afterwards
"""
import torch
import torch.nn as nn

from .utils.quantize import QConv2d, QLinear, QuantConv2d, QuantLinear, QuantNConv2d, QuantNLinear

_CONV_TYPES = (nn.Conv2d, QConv2d, QuantConv2d, QuantNConv2d)
_LINEAR_TYPES = (nn.Linear, QLinear, QuantLinear, QuantNLinear)


def find_prev_bn(bn_module, relu_attached, graph, bottoms, bot):
    """
    Find the batchnorm layers for calculation of expectation or min/max value of input activation.
    And find branching type(one, add, or cat).

    Breadth-first walk from the inputs `bot` of a node back to the nearest registered BatchNorms.  Every
    path carries a branch id string whose first character is the index of the direct input it started
    from and whose length is its depth; a path that crosses an "add"/"cat" node is tagged with that
    connection type (adds followed by an activation are tagged "add_<activation>").
    Returns (bn_list [(module, branch_id)], relu_attach_list, connect_type_list, targ_without_bn).
    """
    queue = [(key, str(i)) for i, key in enumerate(bot)]
    kind = {str(i): 'one' for i in range(len(bot))}
    targ_without_bn = {}
    bn_list, relu_attach_list, connect_type_list = [], [], []
    merged = False                                   # an add/cat was seen anywhere so far (reference: cat_add_found)
    while queue:
        key, bid = queue.pop(0)
        node = graph[key]
        if type(node) == str:
            if 'add' in key:
                kind[bid] = 'add_{}'.format(relu_attached[key]) if key in relu_attached else 'add'
                merged = True
            elif 'cat' in key:
                kind[bid] = 'cat'
                merged = True
        elif not merged and type(node) in _CONV_TYPES + _LINEAR_TYPES:
            print("Warning: {} layer before first batch norm layer detected. The calculated value range might be off.".format(type(node)))
            if bid[0] in targ_without_bn:
                assert False, "Multiple conv/linear layer without batch_norm is not supported."
            targ_without_bn[bid[0]] = ("conv" if type(node) in _CONV_TYPES else "linear", node)

        if key not in bn_module:
            deeper = bid + bid[0]
            queue.extend((src, deeper) for src in bottoms[key])
            kind[deeper] = kind[bid]
        else:
            bn_list.append((bn_module[key], bid))
            relu_attach_list.append(relu_attached[key])
            connect_type_list.append(kind[bid])
    return bn_list, relu_attach_list, connect_type_list, targ_without_bn


def relu_between(graph, bottoms, second, first) -> bool:
    """dfq.py:123-130: whether the walk from `second` back to `first` meets a torch.nn.ReLU (ReLU6 does not count); the
    path must be 1-to-1."""
    key = second
    while key != first:
        assert len(bottoms[key]) == 1, 'graph in equalization relations should be 1-to-1 input-output'
        if type(graph[bottoms[key][0]]) == torch.nn.ReLU:
            return True
        key = bottoms[key][0]
    return False


def merge_order(entries):
    """The order in which dfq.py:228-275 (and layer_transform.py:490-567) folds the BNs of one branch:
    deepest path first, then ties of equal depth, cutting the depth when none is left at the current one.

    entries: list of (branch_id, payload...) tuples; returns the same tuples in processing order.  The
    reference sorts by len(branch_id) descending (stable) and consumes runs of equal depth, which visits the
    sorted list front to back - so the stable sort IS the processing order.
    """
    return sorted(entries, key=lambda e: len(e[0]), reverse=True)


def bias_correction_recipe(graph, bottoms, targ_type, bn_type=torch.nn.BatchNorm2d):
    """One dict per corrected layer, in graph order:

        layer    graph key of the target layer
        terms    [dict(bn=<graph key>, relu=bool, op='set'|'cat'|'add')]  -> E[x] (dfq.py:228-278)
        next_bn  graph key of the BN whose fake_bias gets -delta (dfq.py:204-206, 293) or None
        level    dependency level: a layer reading a fake_bias that an EARLIER layer's delta lands in is at a
                 higher level than that layer; levels are non-decreasing in graph order

    Control flow mirrored from dfq.py:186-216: nodes without bottoms or fed by 'Data' are skipped; BN nodes
    are registered (and consume the pending -delta); a ReLU directly on a registered BN marks it rectified.
    """
    key_of = {}
    bn_module, relu_attached = {}, {}
    recipe = []
    pending = None                                    # index into recipe of the layer whose delta is pending
    for key in graph:
        bot = bottoms[key]
        if bot is None or bot[0] == 'Data':
            continue
        node = graph[key]
        if type(node) == bn_type:
            bn_module[key] = node
            key_of[id(node)] = key
            relu_attached[key] = False
            if pending is not None:
                recipe[pending]["next_bn"] = key
                pending = None
            continue
        if type(node) == torch.nn.ReLU:
            if bot[0] in bn_module:
                relu_attached[bot[0]] = True
        if type(node) in targ_type:
            bn_list, relu_list, type_list, _ = find_prev_bn(bn_module, relu_attached, graph, bottoms, bot[:])
            branches = {}
            for (bn, bid), relu, ctype in zip(bn_list, relu_list, type_list):
                branches.setdefault(bid[0], []).append((bid, key_of[id(bn)], bool(relu), ctype))
            assert len(branches) == 1, "Error while calculating expectation for bias correction"
            ordered = merge_order(list(branches.values())[0])
            terms = []
            for i, (bid, bn_key, relu, ctype) in enumerate(ordered):
                op = 'set' if i == 0 else ('cat' if ctype == 'cat' else 'add')
                terms.append(dict(bn=bn_key, relu=relu, op=op))
            recipe.append(dict(layer=key, terms=terms, next_bn=None, level=0))
            pending = len(recipe) - 1
    # dependency levels
    writer = {}                                       # bn key -> recipe index whose delta lands there
    for i, step in enumerate(recipe):
        if step["next_bn"] is not None:
            writer.setdefault(step["next_bn"], []).append(i)
    level = 0
    for i, step in enumerate(recipe):
        need = level
        for t in step["terms"]:
            for w in writer.get(t["bn"], []):
                if w < i:
                    need = max(need, recipe[w]["level"] + 1)
        level = max(level, need)
        step["level"] = level
    return recipe
