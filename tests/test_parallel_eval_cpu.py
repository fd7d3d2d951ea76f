"""Host side of the partition-parallel evaluation: the ``--parallel-eval`` switch, and the validation / test masks
``data.make_local_partition`` now draws (the papers100M-shape path had nothing to evaluate) without moving a bit of what
it already returned."""
import hashlib

import pytest
import torch

# sha256 prefixes of every tensor make_local_partition(name, rank, 3, seed=1, scale) returned before it drew the masks
PARENT_DIGESTS = {
    ("papers100m", 0): ((7403, 13838), {
        '_ID': 'a5e9a469183d9347', 'feat': '5bf26f841a452a50', 'in_deg': 'dbc3e633d2f64f41',
        'inner_node': '20aba296f48cc554', 'label': '8f25d8b58d8a71bb', 'out_deg': 'dbc3e633d2f64f41',
        'part_id': '7f8c30e1966011a7', 'train_mask': 'b13447be95373ed2', 'indptr': '70f55ca26a8fa79f',
        'indices': '3dcc26f54bc4a11c', 'ranges': 'e8d2877a085c70ee'}),
    ("papers100m", 1): ((7404, 13796), {
        '_ID': 'c7805d20e3080a6c', 'feat': 'b20661cfea568beb', 'in_deg': 'd8b65a6d855c4fa8',
        'inner_node': 'b0b2a94abf1c8308', 'label': '3130726ac9056884', 'out_deg': 'd8b65a6d855c4fa8',
        'part_id': '8ed8c68ccfc98acf', 'train_mask': '22129a07885ba93f', 'indptr': 'e968688a370721e3',
        'indices': '14d73ebccf6d2fdf', 'ranges': 'e8d2877a085c70ee'}),
    ("papers100m", 2): ((7404, 13850), {
        '_ID': '4f0eb1927e30c330', 'feat': '48dff7bad067c18e', 'in_deg': 'ffe69bc2a0734983',
        'inner_node': '58b2d3ad8c8ac77d', 'label': '4b155f3a082bac9f', 'out_deg': 'ffe69bc2a0734983',
        'part_id': '419336045af834c1', 'train_mask': '03746c2aeabd0735', 'indptr': '7b86883d383ee872',
        'indices': '8913841e17b3c118', 'ranges': 'e8d2877a085c70ee'}),
    ("reddit", 0): ((155, 310), {
        '_ID': '864103aebc82aa1b', 'feat': 'a67294c586e5f5ca', 'in_deg': 'd49130e7310c38f5',
        'inner_node': 'a19f642e2ca2ea34', 'label': '543b15e4b7f1e269', 'out_deg': 'd49130e7310c38f5',
        'part_id': 'b8352c62d83d23c0', 'train_mask': 'ed934be1e1524a11', 'indptr': 'b66181b32af826f7',
        'indices': '97c1cc68ee5351d0', 'ranges': '0e7b5de419080052'}),
    ("reddit", 1): ((155, 310), {
        '_ID': '19cd1f525177b78e', 'feat': 'f9e957a17fcd854d', 'in_deg': '3751982de6e86e73',
        'inner_node': 'a19f642e2ca2ea34', 'label': '54a9f214fa2ccd4e', 'out_deg': '3751982de6e86e73',
        'part_id': '53c88bca453cb118', 'train_mask': 'd7254ac07749437f', 'indptr': '018ffc827168e80f',
        'indices': 'f9a5d2d1efd07c9a', 'ranges': '0e7b5de419080052'}),
    ("reddit", 2): ((155, 310), {
        '_ID': '13502c659395040a', 'feat': '8a88d3da1e2fb8d6', 'in_deg': '538e9ccf768754e1',
        'inner_node': 'a19f642e2ca2ea34', 'label': 'b871a2096ea72d79', 'out_deg': '538e9ccf768754e1',
        'part_id': '58012883d0422d83', 'train_mask': 'dd8cfa7dfc0c442e', 'indptr': '9f8dd1d4cceb4b2e',
        'indices': 'edb6859807d53b72', 'ranges': '0e7b5de419080052'}),
}
SCALE = {"papers100m": 0.0002, "reddit": 0.002}


def _digest(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()[:16]


@pytest.mark.parametrize("argv", [["--parallel-eval"], ["--parallel_eval"]])
def test_parallel_eval_switch_parses(argv):
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser(argv).parallel_eval is True


def test_parallel_eval_is_off_by_default():
    from bns_gcn_b200.helper.parser import create_parser
    assert create_parser([]).parallel_eval is False


@pytest.mark.parametrize("name,rank", sorted(PARENT_DIGESTS))
def test_local_partition_masks_leave_the_rest_unchanged(name, rank):
    from bns_gcn_b200.data import SHAPES, make_local_partition
    p = make_local_partition(name, rank, 3, seed=1, device=torch.device("cpu"), scale=SCALE[name])
    (n_in, n_halo), want = PARENT_DIGESTS[(name, rank)]
    assert (p.graph.n_in, p.graph.n_halo) == (n_in, n_halo)
    got = {k: _digest(v) for k, v in p.node_dict.items() if k not in ("val_mask", "test_mask")}
    got.update(indptr=_digest(p.graph.indptr), indices=_digest(p.graph.indices), ranges=_digest(p.gpb.ranges))
    assert got == want
    tr, va, te = p.node_dict["train_mask"], p.node_dict["val_mask"], p.node_dict["test_mask"]
    assert va.dtype == te.dtype == torch.bool and va.shape == te.shape == tr.shape
    assert not (va & tr).any() and not (te & tr).any() and not (va & te).any()
    spec = SHAPES[name]
    if name == "papers100m":                  # ogbn-papers100M's split fractions
        assert (spec["val"], spec["test"]) == (0.0011, 0.0019)
        # ~8 and ~14 nodes of 7,404 expected: only ask that the draw is not empty and not wildly off
        assert 0 < int(va.sum()) + int(te.sum()) < 0.02 * n_in
    else:                                     # make_graph's split of the rest: 1/3 validation, 2/3 test
        assert int(va.sum()) > 0 and int(te.sum()) > int(va.sum())


def test_local_partition_papers100m_split_fractions():
    """At a size where the fractions show: validation and test near ogbn-papers100M's 0.11 % and 0.19 %."""
    from bns_gcn_b200.data import make_local_partition
    p = make_local_partition("papers100m", 0, 1, seed=0, device=torch.device("cpu"), scale=0.003)
    n = p.graph.n_in
    va, te = p.node_dict["val_mask"].double().mean().item(), p.node_dict["test_mask"].double().mean().item()
    assert abs(va - 0.0011) < 5 * (0.0011 / n) ** 0.5 and abs(te - 0.0019) < 5 * (0.0019 / n) ** 0.5, (n, va, te)
