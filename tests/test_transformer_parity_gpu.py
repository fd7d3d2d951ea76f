"""``--model transformer`` training against the CPU oracle (``tests/transformer_oracle.py``: ``TransformerConvRef`` on
the oracle's explicit edge lists, run by its ``OracleRank`` with the exchange unscaled).  The cases are those of
``test_gatv2_training_parity``: P = 1 / 2 / 3, sampling rate 0.3 to 1, 1 and 2 heads, both transports, multi-label BCE
(``tiny-ml``) and single-label CE with 5 classes (a per-head width padded to 8), plus a closing linear layer
(``--n-linear 1``).  Every rank's layer outputs, logits, all-reduced gradients and loss are held to GAT's bar (1e-4
relative), the received index sets are exactly the peers' draws, and so are the weights after the Adam step, with the
exceptions stated below.

The key bias gets no gradient: adding it to every key adds ``<q_v, b_k>`` to every score of row v, which the softmax
ignores (its gradient is ``sum_v q_v sum_u d s_uv`` with ``sum_u d s_uv = 0``).  Both implementations give it rounding
noise, so its gradient is held to be noise (below 1e-5 of the key weight's gradient) rather than to the bar.  Adam's
first step moves every weight by ``lr * g / (|g| + eps)``, so where ``g`` is such noise -- the whole key bias, and any
entry with ``|g| < 1e-4 max |g|`` of its tensor in the oracle's gradient -- the step is anything in ``[-lr, lr]``; those
weights are held to the bound of the step, ``2 lr``, all others to the bar.  For the same reason the run is one epoch:
a second epoch starts from weights that differ by such steps."""
import argparse

import pytest
import torch

from tests.test_parity_gpu import TOL
from tests.transformer_oracle import oracle_kind

pytestmark = pytest.mark.gpu

AMPLIFIED = 1e-4        # |g| / max |g| below which Adam's step is decided by rounding noise


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def _key_bias_indices(args, fg):
    """Positions of the ``lin_key.bias`` tensors in ``model.parameters()``, the order both harnesses list."""
    from bns_gcn_b200 import train
    from bns_gcn_b200.helper.utils import get_layer_size
    a = argparse.Namespace(**vars(args))
    a.n_train = int(fg.train_mask.sum())
    net = train.create_model(get_layer_size(fg.n_feat, a.n_hidden, fg.n_class, a.n_layers), a)
    names = [n for n, _ in net.named_parameters()]
    assert names[names.index("layers.0.lin_key.bias") - 1] == "layers.0.lin_key.weight"
    return {i for i, n in enumerate(names) if n.endswith("lin_key.bias")}


@pytest.mark.parametrize("kw", [
    dict(n_parts=1, sampling_rate=1.0),
    dict(n_parts=2, sampling_rate=1.0, heads=2),
    dict(n_parts=3, sampling_rate=0.5),
    dict(n_parts=3, sampling_rate=0.3, heads=2, backend="p2p", n_layers=3),
    dict(n_parts=2, sampling_rate=0.5, shape="tiny"),
    dict(n_parts=2, sampling_rate=0.5, heads=2, n_layers=3, n_linear=1),
], ids=["p1", "p2-heads2", "p3", "p3-heads2-p2p", "tiny-ce", "p2-n-linear1"])
def test_transformer_training_parity(built, monkeypatch, kw):
    from bns_gcn_b200.data import make_graph, partition_graph
    from tests import harness
    kw = dict(kw)
    shape = kw.pop("shape", "tiny-ml")
    P = kw.pop("n_parts")
    fg = make_graph(shape, seed=0)
    parts = partition_graph(fg, P, "random", seed=0)
    args = harness.make_args(dataset=shape, model="transformer", n_partitions=P, multilabel=(shape == "tiny-ml"),
                             **{"n_layers": 2, **kw})
    key_bias = _key_bias_indices(args, fg)
    prod = harness.run_product(parts, args, "cuda:0", 1)
    selected = [[prod[r]["selected"][0] for r in range(P)]]
    with oracle_kind(monkeypatch):
        orc = harness.run_oracle(parts, args, 1, selected if P > 1 else None)
    for r in range(P):
        for k in list(prod[r]["layers"]) + ["logits", "feat0"]:
            a = prod[r]["layers"][k] if k.startswith("layer") else prod[r][k]
            b = orc[r]["layers"][k] if k.startswith("layer") else orc[r][k]
            assert _rel(a, b) < TOL, (r, k, _rel(a, b))
        assert abs(prod[r]["loss"][0] - orc[r]["loss"][0]) <= 1e-4 * abs(orc[r]["loss"][0]), r
        for i, (a, b) in enumerate(zip(prod[r]["grads"], orc[r]["grads"])):
            if i in key_bias:                           # noise next to the key weight's gradient (listed just before)
                scale = orc[r]["grads"][i - 1].abs().max()
                assert a.abs().max() < 1e-5 * scale and b.abs().max() < 1e-5 * scale, (r, "grad", i)
            else:
                assert _rel(a, b) < TOL, (r, "grad", i, _rel(a, b))
        for i, (a, b, g) in enumerate(zip(prod[r]["params"], orc[r]["params"], orc[r]["grads"])):
            noisy = g.abs() < AMPLIFIED * g.abs().max()
            if i in key_bias:
                noisy = torch.ones_like(noisy)
            diff = (a - b).abs()
            assert diff[~noisy].norm() < TOL * b.norm(), (r, "param", i, (diff[~noisy].norm() / b.norm()).item())
            assert torch.all(diff[noisy] <= 2 * args.lr * (1 + 1e-5)), (r, "param", i)
        for j in range(P):
            if j != r:
                assert torch.equal(prod[j]["one_hops"][0][r], prod[r]["selected"][0][j])
