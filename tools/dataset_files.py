"""Write a ``FullGraph`` in the published layout of Reddit, Yelp or ogbn-products, the files
``bns_gcn_b200.data.load_files`` reads.  ``load_files(write(make_graph(shape)))`` rebuilds the generated graph bit for
bit (for Yelp, with its features standardised), so the readers are checked without downloading anything.

* reddit:  ``reddit_graph.npz`` holds every edge, self-loops included (row = source); the reader replaces the loops.
* yelp:    the same matrix as ``adj_full.npz``; labels as 0 / 1 lists; the features as generated (unscaled).
* products: each undirected pair once, no self-loops: the generated graphs are symmetric with one self-loop per node,
  so the reader's inverse edges and re-added self-loops rebuild them.  Features are written with 9 significant digits,
  which every f32 survives.
"""
from __future__ import annotations

import gzip
import json
import os

import numpy as np

_CSV_ROWS = 8192                     # rows formatted per write


def _adjacency(fg):
    import scipy.sparse as sp
    src, dst = fg.src.numpy(), fg.dst().numpy()
    return sp.coo_matrix((np.ones(src.size, dtype=np.float32), (src, dst)), shape=(fg.n_nodes, fg.n_nodes))


def write_reddit(fg, root: str) -> str:
    import scipy.sparse as sp
    d = os.path.join(root, "reddit")
    os.makedirs(d, exist_ok=True)
    types = np.where(fg.train_mask.numpy(), 1, np.where(fg.val_mask.numpy(), 2, np.where(fg.test_mask.numpy(), 3, 0)))
    np.savez(os.path.join(d, "reddit_data.npz"), feature=fg.feat.numpy(), label=fg.label.numpy(),
             node_types=types.astype(np.int32))
    sp.save_npz(os.path.join(d, "reddit_graph.npz"), _adjacency(fg))
    return d


def write_yelp(fg, root: str) -> str:
    import scipy.sparse as sp
    d = os.path.join(root, "yelp")
    os.makedirs(d, exist_ok=True)
    sp.save_npz(os.path.join(d, "adj_full.npz"), _adjacency(fg))
    np.save(os.path.join(d, "feats.npy"), fg.feat.numpy())
    label = fg.label.numpy().astype(np.int64)
    with open(os.path.join(d, "class_map.json"), "w") as f:
        json.dump({str(i): row for i, row in enumerate(label.tolist())}, f)
    ids = lambda m: np.nonzero(m.numpy())[0].tolist()       # noqa: E731
    with open(os.path.join(d, "role.json"), "w") as f:
        json.dump({"tr": ids(fg.train_mask), "va": ids(fg.val_mask), "te": ids(fg.test_mask)}, f)
    return d


def _write_csv(path: str, a: np.ndarray, fmt: str) -> None:
    """Headerless CSV, one row of ``a`` per line.  Many rows go through one ``%`` so the formatting stays in C."""
    a = a.reshape(a.shape[0], -1)
    line = ",".join([fmt] * a.shape[1]) + "\n"
    with gzip.open(path, "wt", compresslevel=1) as f:
        for i in range(0, a.shape[0], _CSV_ROWS):
            b = a[i:i + _CSV_ROWS]
            f.write((line * b.shape[0]) % tuple(b.ravel().tolist()))


def write_products(fg, root: str) -> str:
    raw = os.path.join(root, "ogbn_products", "raw")
    split = os.path.join(root, "ogbn_products", "split", "sales_ranking")
    os.makedirs(raw, exist_ok=True)
    os.makedirs(split, exist_ok=True)
    src, dst = fg.src.numpy(), fg.dst().numpy()
    once = src < dst
    _write_csv(os.path.join(raw, "edge.csv.gz"), np.stack([src[once], dst[once]], 1), "%d")
    _write_csv(os.path.join(raw, "node-feat.csv.gz"), fg.feat.numpy().astype(np.float64), "%.9g")
    _write_csv(os.path.join(raw, "node-label.csv.gz"), fg.label.numpy(), "%d")
    _write_csv(os.path.join(raw, "num-node-list.csv.gz"), np.array([fg.n_nodes]), "%d")
    for name, m in (("train", fg.train_mask), ("valid", fg.val_mask), ("test", fg.test_mask)):
        _write_csv(os.path.join(split, f"{name}.csv.gz"), np.nonzero(m.numpy())[0], "%d")
    return os.path.join(root, "ogbn_products")


WRITERS = {"reddit": write_reddit, "yelp": write_yelp, "ogbn-products": write_products}


def standard_scaled(fg):
    """``fg`` with its features standardised as the Yelp reader does (``StandardScaler`` fit on the training rows)."""
    import dataclasses

    import torch
    from sklearn.preprocessing import StandardScaler
    scaler = StandardScaler().fit(fg.feat[fg.train_mask].numpy())
    return dataclasses.replace(fg, feat=torch.tensor(scaler.transform(fg.feat.numpy()), dtype=torch.float))
