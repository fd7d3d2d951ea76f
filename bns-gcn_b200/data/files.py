"""Reddit, Yelp and ogbn-products from their published files (``--data-source files``).

The reference's ``load_data`` (``helper/utils.py:37-70``) reads these datasets through DGL and OGB.  This module reads
the raw files those libraries leave under ``--data-path`` after their first run, with numpy / scipy / gzip / json
only, and applies the same rules:

    reddit          reddit/reddit_data.npz     feature [N, F], label [N], node_types [N] (1 train, 2 val, 3 test)
                    reddit/reddit_graph.npz    scipy sparse (``sp.save_npz``), row = source, column = destination
    yelp            yelp/adj_full.npz          scipy sparse, row = source
                    yelp/feats.npy             [N, F]
                    yelp/class_map.json        {"<id>": [0/1, ...]}
                    yelp/role.json             {"tr": [...], "va": [...], "te": [...]}
    ogbn-products   ogbn_products/raw/{edge,node-feat,node-label,num-node-list}.csv.gz        (no header rows)
                    ogbn_products/split/sales_ranking/{train,valid,test}.csv.gz              (one id per line)

* The sparse matrices become edges the way DGL's ``from_scipy`` makes them: every stored entry is one edge, its
  value ignored, duplicates kept.  ogbn-products adds the inverse of every raw edge (OGB's ``add_inverse_edge``).
* Every self-loop is removed and exactly one is added per node (``utils.py:68-69``).  Multi-edges stay: each copy
  counts in the sums and in both degrees, as in DGL.
* Yelp's labels become f32 multi-hot rows, and its features are standardised with a ``StandardScaler`` fit on the
  training rows (``utils.py:45-57``).  ogbn-products' labels are ``view(-1).long()`` (``utils.py:25``).
* ``n_class`` is ``label.max() + 1``, or the label width for multi-label data (``utils.py:62-65``).

Malformed input is refused with ``DataFileError`` naming the file, before anything is built from it.  DGL's ``.bin``
and OGB's ``processed/`` caches are not read.  ogbn-papers100M is refused: its 111 M nodes and 57 GB of features do not
fit the whole-graph partitioner (``make_local_partition`` generates its shape per rank instead).
"""
from __future__ import annotations

import gzip
import json
import os
from typing import Optional

import numpy as np
import torch

from .synthetic import FullGraph, make_graph

DATA_SOURCES = ("synthetic", "files")


class DataFileError(ValueError):
    """A dataset file that is missing or malformed; the message starts with its path."""

    def __init__(self, path: str, what: str):
        super().__init__(f"{path}: {what}")
        self.path = path


def _need(path: str) -> str:
    if not os.path.isfile(path):
        raise DataFileError(path, "no such file")
    return path


def csr_by_destination(n: int, src: torch.Tensor, dst: torch.Tensor, device: torch.device):
    """``dgl.remove_self_loop`` then ``dgl.add_self_loop`` (``utils.py:68-69``) on an edge list, as CSR by destination
    with the sources sorted inside each row -- the sort ``chung_lu_edges`` and ``relabel`` use.  Duplicate edges stay.
    Equal keys are equal (dst, src) pairs, so the result does not depend on the device's sort order."""
    src = src.to(device=device, dtype=torch.int64)
    dst = dst.to(device=device, dtype=torch.int64)
    keep = src != dst
    loops = torch.arange(n, dtype=torch.int64, device=device)
    dst = torch.cat([dst[keep], loops])
    src = torch.cat([src[keep], loops])
    del keep
    order = torch.argsort(dst * n + src)
    dst, src = dst[order], src[order]
    del order
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=device)
    indptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n), 0)
    return indptr.cpu(), src.cpu()


# ---- checks shared by the readers ----------------------------------------------------------------------------------

def _sparse_edges(path: str):
    """(N, src, dst) of a ``sp.save_npz`` matrix, row = source: every stored entry, duplicates included."""
    import scipy.sparse as sp
    try:
        m = sp.load_npz(_need(path))
    except DataFileError:
        raise
    except Exception as e:                                  # a zip without the scipy keys, or not a zip at all
        raise DataFileError(path, f"not a scipy sparse matrix ({e})") from e
    if len(m.shape) != 2 or m.shape[0] != m.shape[1]:
        raise DataFileError(path, f"the adjacency matrix is {m.shape[0]} x {m.shape[1]}, not square")
    coo = m.tocoo()                                         # expands the stored entries; sums nothing
    return int(m.shape[0]), torch.from_numpy(np.asarray(coo.row)), torch.from_numpy(np.asarray(coo.col))


def _check_n(path: str, n: int):
    if n <= 0:
        raise DataFileError(path, "the graph has no nodes")


def _features(path: str, feat: np.ndarray, n: int) -> torch.Tensor:
    if feat.ndim != 2:
        raise DataFileError(path, f"features have shape {tuple(feat.shape)}, not [N, F]")
    if feat.shape[0] != n:
        raise DataFileError(path, f"{feat.shape[0]} feature rows for {n} nodes")
    feat = np.ascontiguousarray(feat, dtype=np.float32)
    bad = ~np.isfinite(feat)
    if bad.any():
        r, c = (int(x[0]) for x in np.nonzero(bad))
        raise DataFileError(path, f"non-finite feature {feat[r, c]} at node {r}, column {c}")
    return torch.from_numpy(feat)


def _class_labels(path: str, label: np.ndarray, n: int) -> torch.Tensor:
    if not np.issubdtype(label.dtype, np.integer):
        raise DataFileError(path, f"labels are {label.dtype}, not integers")
    label = label.reshape(-1)
    if label.size != n:
        raise DataFileError(path, f"{label.size} labels for {n} nodes")
    if label.min() < 0:
        raise DataFileError(path, f"negative label {int(label.min())} at node {int(np.argmin(label))}")
    return torch.from_numpy(label.astype(np.int64))


def _ids(path: str, ids, n: int, what: str) -> torch.Tensor:
    try:
        a = np.asarray(ids)
        if a.size == 0:
            a = a.astype(np.int64)
        if a.ndim != 1 or not np.issubdtype(a.dtype, np.integer):
            raise ValueError(f"{a.dtype} of shape {tuple(a.shape)}")
    except ValueError as e:
        raise DataFileError(path, f"{what} are not a list of node ids ({e})") from e
    if a.size and (a.min() < 0 or a.max() >= n):
        bad = int(a[(a < 0) | (a >= n)][0])
        raise DataFileError(path, f"{what}: node id {bad} outside [0, {n})")
    return torch.from_numpy(a.astype(np.int64))


def _mask(n: int, ids: torch.Tensor) -> torch.Tensor:
    m = torch.zeros(n, dtype=torch.bool)
    m[ids] = True
    return m


def _graph(n, src, dst, feat, label, train, val, test, device) -> FullGraph:
    indptr, src = csr_by_destination(n, src, dst, device)
    n_class = int(label.shape[1]) if label.dim() == 2 else int(label.max()) + 1
    return FullGraph(n, indptr, src, feat, label, train, val, test, n_class)


# ---- the three layouts ---------------------------------------------------------------------------------------------

def _read_reddit(root: str, device) -> FullGraph:
    d = os.path.join(root, "reddit")
    data_path = _need(os.path.join(d, "reddit_data.npz"))
    n, src, dst = _sparse_edges(os.path.join(d, "reddit_graph.npz"))
    _check_n(os.path.join(d, "reddit_graph.npz"), n)
    try:
        data = np.load(data_path, allow_pickle=False)
        keys = set(data.files)
    except Exception as e:
        raise DataFileError(data_path, f"not an .npz archive ({e})") from e
    with data:
        for k in ("feature", "label", "node_types"):
            if k not in keys:
                raise DataFileError(data_path, f"no key {k!r} (it holds {sorted(keys)})")
        feat = _features(data_path, data["feature"], n)
        label = _class_labels(data_path, data["label"], n)
        types = data["node_types"].reshape(-1)
    if types.size != n:
        raise DataFileError(data_path, f"{types.size} node types for {n} nodes")
    types = torch.from_numpy(np.asarray(types))
    return _graph(n, src, dst, feat, label, types == 1, types == 2, types == 3, device)


def _read_json(path: str):
    try:
        with open(_need(path)) as f:
            return json.load(f)
    except DataFileError:
        raise
    except (ValueError, UnicodeDecodeError) as e:
        raise DataFileError(path, f"not JSON ({e})") from e


def _read_yelp(root: str, device) -> FullGraph:
    d = os.path.join(root, "yelp")
    n, src, dst = _sparse_edges(os.path.join(d, "adj_full.npz"))
    _check_n(os.path.join(d, "adj_full.npz"), n)
    feat_path = _need(os.path.join(d, "feats.npy"))
    try:
        feat = np.load(feat_path, allow_pickle=False)
    except Exception as e:
        raise DataFileError(feat_path, f"not an .npy array ({e})") from e
    feat = _features(feat_path, feat, n)

    cm_path = os.path.join(d, "class_map.json")
    cm = _read_json(cm_path)
    if not isinstance(cm, dict):
        raise DataFileError(cm_path, "not a {node id: labels} object")
    if len(cm) != n:
        raise DataFileError(cm_path, f"{len(cm)} entries for {n} nodes")
    try:
        rows = [cm[str(i)] for i in range(n)]
    except KeyError as e:
        raise DataFileError(cm_path, f"no entry for node {e.args[0]}") from e
    try:
        label = np.array(rows)
    except ValueError as e:
        raise DataFileError(cm_path, f"label rows of different widths ({e})") from e
    if label.ndim != 2 or not np.isin(label, (0, 1)).all():
        raise DataFileError(cm_path, "labels are not rows of 0 / 1 entries of one width")
    label = torch.from_numpy(label.astype(np.float32))

    role_path = os.path.join(d, "role.json")
    role = _read_json(role_path)
    if not isinstance(role, dict):
        raise DataFileError(role_path, "not a {'tr' | 'va' | 'te': node ids} object")
    masks = []
    for k in ("tr", "va", "te"):
        if k not in role:
            raise DataFileError(role_path, f"no key {k!r}")
        masks.append(_mask(n, _ids(role_path, role[k], n, f"role {k!r}")))
    train, val, test = masks
    if not train.any():
        raise DataFileError(role_path, "no training nodes (the feature scaling is fit on them)")
    # utils.py:52-56, with the reference's own scaler: fit on the training rows of the f32 features, applied to all
    from sklearn.preprocessing import StandardScaler
    scaler = StandardScaler()
    scaler.fit(feat[train].numpy())
    feat = torch.tensor(scaler.transform(feat.numpy()), dtype=torch.float)
    return _graph(n, src, dst, feat, label, train, val, test, device)


def _read_csv(path: str, dtype, what: str) -> np.ndarray:
    """A headerless comma-separated ``.csv.gz`` as a 2-D array (no rows: shape ``(0, 1)``)."""
    import warnings
    try:
        with gzip.open(_need(path), "rt") as f, warnings.catch_warnings():
            warnings.simplefilter("ignore", UserWarning)          # "input contained no data": checked by the caller
            return np.loadtxt(f, delimiter=",", dtype=dtype, ndmin=2)
    except DataFileError:
        raise
    except (ValueError, OSError, EOFError) as e:
        raise DataFileError(path, f"malformed {what} ({e})") from e


def _read_products(root: str, device) -> FullGraph:
    raw = os.path.join(root, "ogbn_products", "raw")
    split = os.path.join(root, "ogbn_products", "split", "sales_ranking")
    nn_path = os.path.join(raw, "num-node-list.csv.gz")
    nn = _read_csv(nn_path, np.int64, "node count")
    if nn.size != 1:
        raise DataFileError(nn_path, f"{nn.size} node counts; one graph holds one")
    n = int(nn.reshape(-1)[0])
    _check_n(nn_path, n)
    edge_path = os.path.join(raw, "edge.csv.gz")
    edge = _read_csv(edge_path, np.int64, "edge list")
    if edge.shape[0] and edge.shape[1] != 2:
        raise DataFileError(edge_path, f"{edge.shape[1]} columns, not src,dst")
    edge = _ids(edge_path, edge.reshape(-1), n, "edges").view(-1, 2)
    feat_path = os.path.join(raw, "node-feat.csv.gz")
    feat = _features(feat_path, _read_csv(feat_path, np.float32, "features"), n)
    label_path = os.path.join(raw, "node-label.csv.gz")
    label = _read_csv(label_path, np.int64, "labels")
    if label.shape[0] and label.shape[1] != 1:
        raise DataFileError(label_path, f"{label.shape[1]} columns, not one label per node")
    label = _class_labels(label_path, label, n)
    masks = []
    for k in ("train", "valid", "test"):
        p = os.path.join(split, f"{k}.csv.gz")
        ids = _read_csv(p, np.int64, "node ids")
        if ids.shape[0] and ids.shape[1] != 1:
            raise DataFileError(p, f"{ids.shape[1]} columns, not one node id per line")
        masks.append(_mask(n, _ids(p, ids.reshape(-1), n, "split ids")))
    src = torch.cat([edge[:, 0], edge[:, 1]])                # every raw edge and its inverse
    dst = torch.cat([edge[:, 1], edge[:, 0]])
    del edge
    return _graph(n, src, dst, feat, label, *masks, device)


_READERS = {"reddit": _read_reddit, "yelp": _read_yelp, "ogbn-products": _read_products}


def load_files(dataset: str, data_path: str, device: Optional[torch.device] = None) -> FullGraph:
    """``dataset`` read from its published files under ``data_path``, as the ``FullGraph`` ``make_graph`` returns.
    The edges are sorted on ``device`` (default: the GPU when there is one); the CPU builds the identical graph."""
    if dataset in ("ogbn-papers100m", "papers100m"):
        raise ValueError(f"--dataset {dataset} --data-source files: not supported.  The whole-graph partitioner would "
                         "have to hold 111 M nodes and 57 GB of features on one host; papers100M needs per-rank "
                         "loading, which this build only has for the generated shape")
    if dataset not in _READERS:
        raise ValueError(f"--dataset {dataset!r} --data-source files: no published layout is read for it "
                         f"(known: {', '.join(_READERS)})")
    if device is None:
        device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
    return _READERS[dataset](data_path, torch.device(device))


def data_source(args) -> str:
    """``args.data_source``; namespaces made before the flag existed mean the generator."""
    source = getattr(args, 'data_source', 'synthetic')
    if source not in DATA_SOURCES:
        raise ValueError(f"--data-source {source!r}: expected one of {', '.join(DATA_SOURCES)}")
    return source


def load_graph(args, device: Optional[torch.device] = None) -> FullGraph:
    """The whole graph ``args`` names: the seeded generator's shape (``--data-source synthetic``, the default) or the
    dataset's published files under ``--data-path`` (``--data-source files``)."""
    source = data_source(args)
    if source == "files":
        return load_files(args.dataset, args.data_path, device)
    return make_graph(args.dataset, seed=getattr(args, 'graph_seed', 0), device=device)
