"""``ops.plan_col_blocks`` at the dataset shapes of ``data/synthetic.py``, on one partition (the whole graph): the
Reddit shape's F = 256 and F = 128 aggregations run as 2 source-row blocks, narrow passes and low-degree graphs as one,
and ``BNS_SPMM_COLBLOCKS`` overrides the plan."""
import types

import pytest


def _whole_graph(name):
    from bns_gcn_b200.data.synthetic import SHAPES
    s = SHAPES[name]
    return types.SimpleNamespace(n_rows=s["n"], n_cols=s["n"], nnz=s["e"])


@pytest.mark.parametrize("name,F,want", [
    ("reddit", 256, 2), ("reddit", 128, 2), ("reddit", 44, 1), ("reddit", 127, 1),
    ("ogbn-products", 256, 1),          # average degree ~50 < BLOCK_MIN_AVG_DEGREE
    ("ogbn-products", 128, 1),
    ("yelp", 256, 1),
])
def test_plan_col_blocks_at_dataset_shapes(built, monkeypatch, name, F, want):
    from bns_gcn_b200 import ops
    monkeypatch.delenv("BNS_SPMM_COLBLOCKS", raising=False)
    assert ops.plan_col_blocks(_whole_graph(name), F) == want


def test_reddit_blocks_fit_the_table_budget(built):
    """Each of the 2 Reddit-shape blocks holds at most ``BLOCK_TABLE_BYTES`` of 128-float source rows; one would not."""
    from bns_gcn_b200 import ops
    g = _whole_graph("reddit")
    assert g.n_cols * 512 > ops.BLOCK_TABLE_BYTES
    assert -(-g.n_cols // 2) * 512 <= ops.BLOCK_TABLE_BYTES


@pytest.mark.parametrize("forced", ["1", "3", "4"])
def test_env_override_wins(built, monkeypatch, forced):
    from bns_gcn_b200 import ops
    monkeypatch.setenv("BNS_SPMM_COLBLOCKS", forced)
    for name in ("reddit", "ogbn-products", "yelp"):
        for F in (256, 128, 44):
            assert ops.plan_col_blocks(_whole_graph(name), F) == int(forced)
