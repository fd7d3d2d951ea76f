"""On-disk partition store: ``graph_partition`` / ``load_partition`` of the reference (helper/utils.py:73-140).

The reference hands both jobs to DGL (``dgl.distributed.partition_graph`` writes ``<graph_name>.json`` plus one binary
blob per part, ``dgl.distributed.load_partition`` reads one part back); neither DGL nor its file format exists here.
This module keeps the *call contract* -- same function names, same ``args`` fields (``part_path``, ``graph_name``,
``n_partitions``, ``partition_method``, ``inductive``), the same "partition once, skip when the config file exists"
rule (utils.py:86), the same ``meta.json`` with ``n_feat / n_class / n_train`` (utils.py:97-98), and the same return
value ``(subg, node_dict, gpb)`` that ``train.run`` consumes -- over a format made for large parts:

    <part_path>/<graph_name>/<graph_name>.json     part config: counts, node ranges, per-part array table
    <part_path>/<graph_name>/meta.json             {"n_feat": .., "n_class": .., "n_train": ..}
    <part_path>/<graph_name>/part<r>/<key>.npy     one plain ``.npy`` per array (CSR + node_dict entries)

Every array is its own ``.npy`` so a rank maps only what it needs (``np.load(mmap_mode='r')``) and copies it
straight to its GPU; boolean masks are stored as uint8 and cast back on load, exactly the wart the reference
documents for DGL's format (utils.py:85, :114-127).  Local column ids are stored as int32 when they fit (they do up
to 2^31 local nodes) and widened on load (the partition contract is int64).
"""
from __future__ import annotations

import json
import os
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from .partition import NID, GraphPartitionBook, LocalGraph, Partition, partition_graph
from .files import data_source, load_graph
from .synthetic import FullGraph

FORMAT_VERSION = 1
_BOOL_KEYS = ("inner_node", "train_mask", "val_mask", "test_mask")


def partition_balance(args) -> str:
    """``--partition-balance``; an ``args`` built without the field balances node counts."""
    return getattr(args, 'partition_balance', 'nodes')


def default_graph_name(args) -> str:
    """main.py:17-23 of the reference.  A graph read with ``--data-source files`` gets a ``files`` token after the
    dataset (``reddit-files-2-metis-vol-induc``), so that its store is never taken for the generated shape's; an
    edge-balanced partition gets an ``edges`` token after the objective (``reddit-4-metis-vol-edges-induc``)."""
    dataset = args.dataset + ('-files' if data_source(args) == 'files' else '')
    obj = getattr(args, 'partition_obj', 'vol') + ('-edges' if partition_balance(args) == 'edges' else '')
    return '%s-%d-%s-%s-%s' % (dataset, args.n_partitions, args.partition_method, obj,
                               'induc' if args.inductive else 'trans')


def _dirs(args) -> Tuple[str, str]:
    if not getattr(args, 'graph_name', ''):
        args.graph_name = default_graph_name(args)
    graph_dir = os.path.join(args.part_path, args.graph_name)
    return graph_dir, os.path.join(graph_dir, args.graph_name + '.json')


def _check_source(cfg: dict, args, part_config: str) -> None:
    """Refuse a store built from the other ``--data-source`` (a config without the key was generated)."""
    stored, wanted = cfg.get("data_source", "synthetic"), data_source(args)
    if stored != wanted:
        raise RuntimeError(f"{part_config} was partitioned from --data-source {stored}, this run reads --data-source "
                           f"{wanted}; pick another --graph-name or remove the store")


def _check_balance(cfg: dict, args, part_config: str) -> None:
    """Refuse a store partitioned under the other ``--partition-balance`` (a config without the key balanced nodes)."""
    stored, wanted = cfg.get("balance", "nodes"), partition_balance(args)
    if stored != wanted:
        raise RuntimeError(f"{part_config} was partitioned with --partition-balance {stored}, this run asks for "
                           f"--partition-balance {wanted}; pick another --graph-name or remove the store")


def _save_array(path: str, t: torch.Tensor) -> Dict[str, object]:
    a = t.detach().cpu().contiguous().numpy()
    if a.dtype == np.bool_:
        a = a.astype(np.uint8)
    np.save(path, a, allow_pickle=False)
    return {"dtype": str(a.dtype), "shape": list(a.shape)}


def save_partition(p: Partition, graph_dir: str) -> Dict[str, object]:
    """Write one part; returns its entry of the part config."""
    d = os.path.join(graph_dir, f"part{p.rank}")
    os.makedirs(d, exist_ok=True)
    arrays: Dict[str, object] = {}
    idx = p.graph.indices
    if p.graph.num_nodes() < 2 ** 31:
        idx = idx.to(torch.int32)
    arrays["indptr"] = _save_array(os.path.join(d, "indptr.npy"), p.graph.indptr)
    arrays["indices"] = _save_array(os.path.join(d, "indices.npy"), idx)
    for k, v in p.node_dict.items():
        arrays["node/" + k] = _save_array(os.path.join(d, f"node_{k}.npy"), v)
    return {"dir": f"part{p.rank}", "n_in": p.graph.n_in, "n_halo": p.graph.n_halo, "n_edges": p.graph.num_edges(),
            "arrays": arrays}


def graph_partition(args, fg: Optional[FullGraph] = None, device: Optional[torch.device] = None) -> str:
    """helper/utils.py:73-98: build the graph (``load_data`` -> ``load_graph``: the seeded generator, or the published
    files with ``--data-source files``), partition it unless the part config already exists, always (re)write
    ``meta.json``.  Returns the part-config path.  Nothing is written before the graph is built and checked."""
    graph_dir, part_config = _dirs(args)
    if os.path.exists(part_config):
        with open(part_config) as f:
            cfg = json.load(f)
        _check_source(cfg, args, part_config)
        _check_balance(cfg, args, part_config)
    if fg is None:
        fg = load_graph(args, device)
    n_feat, n_class = fg.n_feat, fg.n_class
    n_train = int(fg.train_mask.sum())                     # utils.py:81 (after the inductive subgraph: the same count)
    os.makedirs(graph_dir, exist_ok=True)
    if not os.path.exists(part_config):                    # utils.py:86
        parts = partition_graph(fg, args.n_partitions, args.partition_method, seed=getattr(args, 'graph_seed', 0),
                                inductive=args.inductive, device=device,
                                objective=getattr(args, 'partition_obj', 'vol'), balance=partition_balance(args))
        cfg = {"format_version": FORMAT_VERSION, "graph_name": args.graph_name, "data_source": data_source(args),
               "num_parts": args.n_partitions, "part_method": args.partition_method, "inductive": bool(args.inductive),
               "balance": partition_balance(args),
               "node_map": [int(x) for x in parts[0].gpb.ranges.tolist()],
               "num_nodes": int(parts[0].gpb.ranges[-1]), "num_edges": int(sum(p.graph.num_edges() for p in parts))}
        for p in parts:
            cfg[f"part-{p.rank}"] = save_partition(p, graph_dir)
        tmp = part_config + ".tmp"
        with open(tmp, 'w') as f:
            json.dump(cfg, f, indent=1)
        os.replace(tmp, part_config)                       # the config appears only when every part is complete
    with open(os.path.join(graph_dir, 'meta.json'), 'w') as f:
        json.dump({'n_feat': n_feat, 'n_class': n_class, 'n_train': n_train}, f)
    return part_config


def _load_array(path: str, mmap: bool) -> torch.Tensor:
    a = np.load(path, mmap_mode='r' if mmap else None, allow_pickle=False)
    return torch.from_numpy(np.array(a))        # a private, writable copy (the mapping itself is read-only)


def load_partition(args, rank: int, device: Optional[torch.device] = None, mmap: bool = True):
    """helper/utils.py:101-140: ``(subg, node_dict, gpb)`` of part ``rank``; fills ``args.n_feat / n_class / n_train``
    from ``meta.json``.  ``device``: where the tensors go (default: stay on the host)."""
    graph_dir, part_config = _dirs(args)
    if not os.path.exists(part_config):
        raise FileNotFoundError(f"{part_config}: no such partition config; run graph_partition(args) first "
                                "(main.py does unless --skip-partition)")
    print('loading partitions')
    with open(part_config) as f:
        cfg = json.load(f)
    if cfg.get("format_version") != FORMAT_VERSION:
        raise RuntimeError(f"{part_config}: format version {cfg.get('format_version')} != {FORMAT_VERSION}")
    _check_source(cfg, args, part_config)
    _check_balance(cfg, args, part_config)
    if not 0 <= rank < cfg["num_parts"]:
        raise IndexError(f"part {rank} of {cfg['num_parts']}")
    if cfg["num_parts"] != args.n_partitions:
        raise RuntimeError(f"{part_config} holds {cfg['num_parts']} parts, --n-partitions is {args.n_partitions}")
    ent = cfg[f"part-{rank}"]
    d = os.path.join(graph_dir, ent["dir"])

    def get(name: str, key: str) -> torch.Tensor:
        t = _load_array(os.path.join(d, name), mmap)
        want = ent["arrays"][key]
        if list(t.shape) != want["shape"] or str(t.numpy().dtype) != want["dtype"]:
            raise RuntimeError(f"{os.path.join(d, name)}: {tuple(t.shape)} {t.numpy().dtype} does not match the part "
                               f"config ({want['shape']} {want['dtype']})")
        return t

    indptr = get("indptr.npy", "indptr").to(torch.int64)
    indices = get("indices.npy", "indices").to(torch.int64)
    node_dict: Dict[str, torch.Tensor] = {}
    for key in ent["arrays"]:
        if not key.startswith("node/"):
            continue
        k = key[5:]
        t = get(f"node_{k}.npy", key)
        if k in _BOOL_KEYS:
            t = t.bool()                                   # utils.py:114, :121, :127-128
        node_dict[k] = t
    if device is not None:
        indptr, indices = indptr.to(device), indices.to(device)
        node_dict = {k: v.to(device) for k, v in node_dict.items()}
    subg = LocalGraph(int(ent["n_in"]), int(ent["n_halo"]), indptr, indices)
    gpb = GraphPartitionBook(torch.tensor(cfg["node_map"], dtype=torch.int64))
    with open(os.path.join(graph_dir, 'meta.json')) as f:
        meta = json.load(f)
    args.n_feat, args.n_class, args.n_train = meta['n_feat'], meta['n_class'], meta['n_train']   # utils.py:134-138
    return subg, node_dict, gpb


def load_as_partition(args, rank: int, device: Optional[torch.device] = None) -> Partition:
    """The same part wrapped as the in-memory ``Partition`` record the tests and tools pass around."""
    subg, nd, gpb = load_partition(args, rank, device)
    return Partition(rank, gpb.num_partitions(), subg, nd, gpb,
                     {"n_feat": args.n_feat, "n_class": args.n_class, "n_train": args.n_train})
