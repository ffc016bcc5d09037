"""CHECKER for the synthetic stack (BASELINE configs[4]): one Conv[C,C,k,k]+BN+ReLU -> Conv[C,C,k,k]+BN block through the
oracle - BN fold (layer_transform.py:246-272), equalization to convergence (dfq.py:78-117), bias correction of the second
conv (dfq.py:173-293) - compared with what the device left in the arena.

Test infrastructure, like everything under oracle/: used by tests/test_gpu_engine.py and by bench.py's `parity_check`
(which verifies blocks of the very stack it timed).  Never on the product path.
"""
import numpy as np

from . import dfq_oracle as O


def oracle_block(before, _pre_correction=None):
    """`before`: [conv1, conv2] dicts of DeviceStack.block_arrays (pristine state).  Returns (layers, bns, sweeps).
    `_pre_correction`: a list that receives the second conv's equalized bias and fake_bias before the correction."""
    layers, bns = [], []
    for d in before:
        w2, b2, fw, fb = O.bn_fold(d["w"], d["bias"], d["gamma"], d["beta"], d["mean"], d["var"], 1e-5)
        layers.append(O.OLayer(w2, b2)); bns.append((fw, fb))
    n, _ = O.cross_layer_equalization(layers, bns, [O.ORelation(0, 1, 0)])
    if _pre_correction is not None:
        _pre_correction += [layers[1].b.copy(), bns[1][1].copy()]
    delta = O.bias_delta(layers[1].w, O.relu_expectation(*bns[0]))
    layers[1].b = layers[1].b + (-delta)
    bns[1] = (bns[1][0], bns[1][1] + (-delta))
    return layers, bns, n


def compare_block(before, after):
    """Returns dict(sweeps, weights_bit_exact, vectors_bit_exact, bias_normwise, bias_rows_outside_bound): the device's block
    `after` vs the oracle run on `before`.  Weights, the first conv's bias and BN vectors are pure equalization outputs (bit-exact
    contract); the second conv's bias and fake_bias carry the bias correction (1e-5 normwise contract; row by row, the number
    of entries whose correction leaves dfq_oracle.bias_delta_bound, widened by the rounding of the bias update)."""
    pre = []
    layers, bns, n = oracle_block(before, pre)
    w_ok = all(np.array_equal(a["w"].reshape(l.w.shape), l.w) for a, l in zip(after, layers))
    v_ok = (np.array_equal(after[0]["bias"], layers[0].b) and np.array_equal(after[0]["fake_w"], bns[0][0])
            and np.array_equal(after[0]["fake_b"], bns[0][1]) and np.array_equal(after[1]["fake_w"], bns[1][0]))
    nw = lambda a, b: float(np.abs(a.astype(np.float64) - b).max() / max(np.abs(b).max(), 1e-30))
    # row by row: bias - delta with delta within bias_delta_bound of the exact value, plus the rounding of that one fp32 add
    eq_w = layers[1].w if w_ok else after[1]["w"].reshape(layers[1].w.shape)
    exact, bound = O.bias_delta_bound(eq_w, O.relu_expectation(*bns[0]))
    out_rows = 0
    for got, base in zip((after[1]["bias"], after[1]["fake_b"]), pre):
        want = base.astype(np.float64) - exact
        out_rows += int(np.count_nonzero(~(np.abs(got.astype(np.float64) - want) <= bound + 2.0 ** -24 * np.abs(want) * (1 + 2.0 ** -20))))
    return dict(sweeps=int(n), weights_bit_exact=bool(w_ok), vectors_bit_exact=bool(v_ok),
                bias_normwise=max(nw(after[1]["bias"], layers[1].b), nw(after[1]["fake_b"], bns[1][1])),
                bias_rows_outside_bound=out_rows)
