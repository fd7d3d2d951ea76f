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
    <part_path>/<graph_name>/{val,test}/...        inductive runs with ``--eval --parallel-eval``: the same layout for
                                                   a partition of each evaluation graph (``load_eval_partition``)

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

from .partition import (NID, GraphPartitionBook, LocalGraph, Partition, induced_subgraph, partition_graph, random_parts,
                        relabel_ids)
from .files import data_source, is_papers100m, load_graph, read_papers100m
from .synthetic import FullGraph, make_local_partition

FORMAT_VERSION = 1
_BOOL_KEYS = ("inner_node", "train_mask", "val_mask", "test_mask")
EVAL_GRAPHS = ("val", "test")


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


def _write_parts(parts, graph_dir: str, part_config: str, cfg: dict) -> None:
    """Write every part, then the part config (through a temporary file: the config appears only when every part is
    complete)."""
    os.makedirs(graph_dir, exist_ok=True)
    for p in parts:
        cfg[f"part-{p.rank}"] = save_partition(p, graph_dir)
    tmp = part_config + ".tmp"
    with open(tmp, 'w') as f:
        json.dump(cfg, f, indent=1)
    os.replace(tmp, part_config)


def _head(args, ranges: torch.Tensor, n_edges: int) -> dict:
    return {"format_version": FORMAT_VERSION, "graph_name": args.graph_name, "data_source": data_source(args),
            "num_parts": args.n_partitions, "part_method": args.partition_method, "inductive": bool(args.inductive),
            "balance": partition_balance(args),
            "node_map": [int(x) for x in ranges.tolist()], "num_nodes": int(ranges[-1]), "num_edges": int(n_edges)}


def _config_head(args, parts) -> dict:
    return _head(args, parts[0].gpb.ranges, sum(p.graph.num_edges() for p in parts))


def _write_meta(graph_dir: str, n_feat: int, n_class: int, n_train: int) -> None:
    with open(os.path.join(graph_dir, 'meta.json'), 'w') as f:
        json.dump({'n_feat': n_feat, 'n_class': n_class, 'n_train': n_train}, f)


def wants_eval_partitions(args) -> bool:
    """``--eval --parallel-eval --inductive``: every rank evaluates its own part of the two evaluation graphs."""
    return bool(getattr(args, 'eval', False) and getattr(args, 'parallel_eval', False) and args.inductive)


def _eval_dirs(args, which: str) -> Tuple[str, str]:
    if which not in EVAL_GRAPHS:
        raise ValueError(f"evaluation graph {which!r}: expected one of {', '.join(EVAL_GRAPHS)}")
    graph_dir, _ = _dirs(args)
    d = os.path.join(graph_dir, which)
    return d, os.path.join(d, args.graph_name + '.json')


def _check_eval(cfg: dict, args, which: str, part_config: str) -> None:
    """Refuse an evaluation set of another graph, source, balance, method or part count."""
    _check_source(cfg, args, part_config)
    _check_balance(cfg, args, part_config)
    for key, stored, wanted in (("eval_graph", cfg.get("eval_graph"), which),
                                ("--partition-method", cfg.get("part_method"), args.partition_method),
                                ("--n-partitions", cfg.get("num_parts"), args.n_partitions)):
        if stored != wanted:
            raise RuntimeError(f"{part_config} was partitioned with {key} {stored}, this run asks for {key} {wanted}; "
                               "pick another --graph-name or remove the store")


def eval_graph_of(fg: FullGraph, which: str) -> FullGraph:
    """The graph an inductive run evaluates on: ``val`` -> the train | val subgraph, ``test`` -> the full graph
    (the reference's ``val_g`` / ``test_g``, helper/utils.py:226-230)."""
    return induced_subgraph(fg, fg.train_mask | fg.val_mask) if which == 'val' else fg


def eval_partitions(fg: FullGraph, which: str, args, device: Optional[torch.device] = None):
    """``partition_graph`` of ``eval_graph_of(fg, which)`` with the run's method, objective, balance and seed.  Each
    part keeps what its evaluation reads: ids and owners, ``feat``, ``label``, the degrees of THAT graph, and the mask
    it is scored on (``val_mask`` / ``test_mask``)."""
    parts = partition_graph(eval_graph_of(fg, which), args.n_partitions, args.partition_method,
                            seed=getattr(args, 'graph_seed', 0), device=device,
                            objective=getattr(args, 'partition_obj', 'vol'), balance=partition_balance(args))
    keep = (NID, "part_id", "inner_node", "feat", "label", "in_deg", "out_deg", which + "_mask")
    for p in parts:
        p.node_dict = {k: p.node_dict[k] for k in keep}
    return parts


def graph_partition(args, fg: Optional[FullGraph] = None, device: Optional[torch.device] = None) -> str:
    """helper/utils.py:73-98: build the graph (``load_data`` -> ``load_graph``: the seeded generator, or the published
    files with ``--data-source files``), partition it unless the part config already exists, always (re)write
    ``meta.json``.  Returns the part-config path.  Nothing is written before the graph is built and checked.
    With ``--eval --parallel-eval --inductive`` the two evaluation sets (``val/``, ``test/``: ``eval_partitions``) are
    written too, each unless its own config exists, from the same ``FullGraph``.
    ogbn-papers100M (``--dataset ogbn-papers100m``) is never built whole: ``papers100m_partition`` writes its store."""
    if fg is None and is_papers100m(args.dataset):
        return papers100m_partition(args, device)
    graph_dir, part_config = _dirs(args)
    if os.path.exists(part_config):
        with open(part_config) as f:
            cfg = json.load(f)
        _check_source(cfg, args, part_config)
        _check_balance(cfg, args, part_config)
    todo = []
    if wants_eval_partitions(args):
        for which in EVAL_GRAPHS:
            _, eval_config = _eval_dirs(args, which)
            if os.path.exists(eval_config):
                with open(eval_config) as f:
                    _check_eval(json.load(f), args, which, eval_config)
            else:
                todo.append(which)
    if fg is None:
        fg = load_graph(args, device)
    n_feat, n_class = fg.n_feat, fg.n_class
    n_train = int(fg.train_mask.sum())                     # utils.py:81 (after the inductive subgraph: the same count)
    os.makedirs(graph_dir, exist_ok=True)
    if not os.path.exists(part_config):                    # utils.py:86
        parts = partition_graph(fg, args.n_partitions, args.partition_method, seed=getattr(args, 'graph_seed', 0),
                                inductive=args.inductive, device=device,
                                objective=getattr(args, 'partition_obj', 'vol'), balance=partition_balance(args))
        _write_parts(parts, graph_dir, part_config, _config_head(args, parts))
        del parts
    for which in todo:
        eval_dir, eval_config = _eval_dirs(args, which)
        parts = eval_partitions(fg, which, args, device)
        cfg = _config_head(args, parts)
        cfg["inductive"], cfg["eval_graph"] = False, which     # a partition of the whole evaluation graph
        _write_parts(parts, eval_dir, eval_config, cfg)
        del parts
    _write_meta(graph_dir, n_feat, n_class, n_train)
    return part_config


# ---- ogbn-papers100M: the store written without the whole graph ---------------------------------------------------

PAPERS_CHUNK = 1 << 21          # edges, or feature rows, read per step: 32 MB of edge ids, 1 GB of 128-wide f32 rows


def papers100m_refusals(args) -> list:
    """Every reason ``args`` cannot train ogbn-papers100M, which is only ever partitioned by streaming (empty: none)."""
    why = []
    if args.partition_method != 'random':
        why.append(f"--partition-method {args.partition_method} partitions the whole graph; only random streams")
    if partition_balance(args) == 'edges':
        why.append("--partition-balance edges swaps nodes by in-degree, which would need the degrees before the "
                   "relabelling pass")
    if args.inductive:
        why.append("--inductive needs the train | val subgraph and a whole-graph evaluation set (the reference runs "
                   "papers100M transductively)")
    if getattr(args, 'eval', False) and not getattr(args, 'parallel_eval', False):
        why.append("--eval without --parallel-eval evaluates on rank 0's whole graph; pass --parallel-eval or --no-eval")
    return why


def check_papers100m(args) -> None:
    """Raise ``ValueError`` naming every reason of ``papers100m_refusals`` (nothing for the other datasets)."""
    why = papers100m_refusals(args) if is_papers100m(args.dataset) else []
    if why:
        raise ValueError(f"--dataset {args.dataset}: " + "; ".join(why))


def _finish(graph_dir: str, part_config: str, cfg: dict, meta) -> None:
    """``meta.json``, then the part config through a temporary file: a store without a config is incomplete."""
    _write_meta(graph_dir, *meta)
    tmp = part_config + ".tmp"
    with open(tmp, 'w') as f:
        json.dump(cfg, f, indent=1)
    os.replace(tmp, part_config)


def _generated_papers(args, graph_dir: str, part_config: str, device) -> None:
    """The generated papers100M shape: part r is ``make_local_partition`` of rank r, one part at a time."""
    entries, n_edges, p = {}, 0, None
    for r in range(args.n_partitions):
        p = make_local_partition("papers100m", r, args.n_partitions, seed=getattr(args, 'graph_seed', 0),
                                 device=device, scale=getattr(args, 'graph_scale', 1.0))
        entries[f"part-{r}"] = save_partition(p, graph_dir)
        n_edges += p.graph.num_edges()
    cfg = _head(args, p.gpb.ranges, n_edges)
    cfg.update(entries)
    _finish(graph_dir, part_config, cfg, (p.meta["n_feat"], p.meta["n_class"], p.meta["n_train"]))


def _spill_edges(pf, new_id, ranges, spills, dev, chunk: int):
    """The edge pass: drop self-loops, map both ends to new ids, count the in- and out-degrees, and append every
    (destination, source) pair, as int64, to the spill file of its destination's part."""
    n, n_parts = pf.n, len(spills)
    in_cnt = torch.zeros(n, dtype=torch.int64, device=dev)
    out_cnt = torch.zeros(n, dtype=torch.int64, device=dev)
    ranges_d = ranges.to(dev)
    for src, dst in pf.edges(chunk):
        s, d = torch.from_numpy(src).to(dev), torch.from_numpy(dst).to(dev)
        keep = s != d
        s, d = new_id[s[keep]], new_id[d[keep]]
        ones = torch.ones(s.numel(), dtype=torch.int64, device=dev)
        out_cnt.index_add_(0, s, ones)
        in_cnt.index_add_(0, d, ones)
        pairs = torch.stack([d, s], 1)
        if n_parts > 1:
            owner = torch.searchsorted(ranges_d, d, right=True) - 1
            pairs = pairs[torch.argsort(owner, stable=True)]
            counts = torch.bincount(owner, minlength=n_parts).tolist()
        else:
            counts = [pairs.shape[0]]
        pairs = pairs.cpu().numpy()
        at = 0
        for f, c in zip(spills, counts):
            if c:
                f.write(memoryview(pairs[at:at + c]))
                at += c
    return in_cnt.cpu(), out_cnt.cpu()


def _streamed_part(pf, r: int, ranges, order, in_cnt, out_cnt, spill_path: str, part_dir: str, dev):
    """Part ``r`` from its spill file, written as ``save_partition`` writes ``extract_partition``'s piece; the feature
    file is created at its size with its header, and filled later by ``_stream_features``."""
    n = pf.n
    start, end = int(ranges[r]), int(ranges[r + 1])
    n_in = end - start
    pairs = torch.from_numpy(np.fromfile(spill_path, dtype=np.int64).reshape(-1, 2)).to(dev)
    loops = torch.arange(start, end, dtype=torch.int64, device=dev)
    dst, src = torch.cat([pairs[:, 0], loops]), torch.cat([pairs[:, 1], loops])
    del pairs
    perm = torch.argsort(dst * n + src)                    # relabel's sort; equal keys are equal pairs
    dst, src = dst[perm], src[perm]
    del perm
    indptr = torch.zeros(n_in + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(torch.bincount(dst - start, minlength=n_in), 0)
    del dst
    inner = (src >= start) & (src < end)
    halo = torch.unique(src[~inner])                       # as extract_partition
    local = torch.where(inner, src - start, n_in + torch.searchsorted(halo, src))
    del src, inner
    n_halo = int(halo.numel())
    if n_in + n_halo < 2 ** 31:
        local = local.to(torch.int32)
    gid = torch.cat([loops, halo])
    part_id = torch.searchsorted(ranges.to(dev), gid, right=True) - 1
    inner_node = torch.zeros(gid.numel(), dtype=torch.bool)
    inner_node[:n_in] = True
    old = order[start:end].cpu().numpy()
    os.makedirs(part_dir, exist_ok=True)
    arrays: Dict[str, object] = {}
    arrays["indptr"] = _save_array(os.path.join(part_dir, "indptr.npy"), indptr)
    arrays["indices"] = _save_array(os.path.join(part_dir, "indices.npy"), local)
    n_edges = int(local.numel())
    del indptr, local
    feat_path = os.path.join(part_dir, "node_feat.npy")
    m = np.lib.format.open_memmap(feat_path, mode="w+", dtype=np.float32, shape=(n_in, pf.n_feat))
    del m
    nd = {NID: gid, "part_id": part_id, "inner_node": inner_node, "feat": None,
          "label": torch.from_numpy(pf.label[old]), "in_deg": in_cnt[start:end] + 1, "out_deg": out_cnt[start:end] + 1,
          "train_mask": torch.from_numpy(pf.train[old]), "val_mask": torch.from_numpy(pf.val[old]),
          "test_mask": torch.from_numpy(pf.test[old])}
    for k, v in nd.items():
        arrays["node/" + k] = ({"dtype": "float32", "shape": [n_in, pf.n_feat]} if v is None else
                               _save_array(os.path.join(part_dir, f"node_{k}.npy"), v))
    return {"dir": os.path.basename(part_dir), "n_in": n_in, "n_halo": n_halo, "n_edges": n_edges, "arrays": arrays}


def _stream_features(pf, part: torch.Tensor, n_in, graph_dir: str, chunk: int) -> None:
    """Every feature row to its part's file (``n_in``: the row count of each).  ``relabel`` keeps each part's nodes in
    their old order, so each part's rows arrive in file order: every file is appended to, after its header."""
    n_parts = len(n_in)
    files = []
    try:
        for r in range(n_parts):
            path = os.path.join(graph_dir, f"part{r}", "node_feat.npy")
            f = open(path, "r+b")
            files.append(f)
            f.seek(os.path.getsize(path) - n_in[r] * pf.n_feat * 4)
        part = part.numpy()
        at = 0
        for rows in pf.features(chunk):
            k = rows.shape[0]
            owner = part[at:at + k]
            at += k
            if n_parts == 1:
                files[0].write(memoryview(rows))
                continue
            rows = rows[np.argsort(owner, kind="stable")]
            bounds = np.cumsum(np.bincount(owner, minlength=n_parts)).tolist()
            for r in range(n_parts):
                lo = bounds[r - 1] if r else 0
                if bounds[r] > lo:
                    files[r].write(memoryview(rows[lo:bounds[r]]))
    finally:
        for f in files:
            f.close()


def papers100m_partition(args, device: Optional[torch.device] = None, chunk: int = PAPERS_CHUNK) -> str:
    """``graph_partition`` for ogbn-papers100M: the store ``partition_graph(fg, P, 'random')`` + ``_write_parts`` would
    write, byte for byte, without ever holding the whole graph.  Returns the part-config path; a store whose config
    exists is kept as it is.

    * ``--data-source files``: the checked node tables (``files.read_papers100m``), the owners ``random_parts`` and
      the ids ``relabel_ids`` give; one pass over the edges (``chunk`` at a time, on ``device``: default the GPU
      when there is one) counts the degrees and spills every edge to its destination's part under a temporary
      directory in the store; then each part is sorted and written in turn; then the feature rows are streamed to
      their parts, ``chunk`` rows at a time.  Host memory: the node tables (a few length-N arrays), one part's
      largest array, and a few chunks -- nothing proportional to E or to N x F.
    * ``--data-source synthetic``: part r is ``make_local_partition('papers100m', r, P, seed=args.graph_seed,
      scale=args.graph_scale)``, the generator ``bench.py`` uses (its ``out_deg`` is its ``in_deg``, and ``n_train``
      comes from the shape's fraction).
    The part config is written last; a failure removes the spill directory, and the store directory when this call
    created it."""
    import shutil
    import tempfile
    check_papers100m(args)
    graph_dir, part_config = _dirs(args)
    if os.path.exists(part_config):
        with open(part_config) as f:
            cfg = json.load(f)
        _check_source(cfg, args, part_config)
        _check_balance(cfg, args, part_config)
        return part_config
    if device is None:
        device = torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")
    dev = torch.device(device)
    pf = read_papers100m(args.data_path) if data_source(args) == "files" else None
    created = not os.path.isdir(graph_dir)
    os.makedirs(graph_dir, exist_ok=True)
    spill_dir = None
    try:
        if pf is None:
            _generated_papers(args, graph_dir, part_config, dev)
            return part_config
        n_parts = args.n_partitions
        part = random_parts(pf.n, n_parts, getattr(args, 'graph_seed', 0))
        order, new_id, ranges = relabel_ids(part, n_parts, dev)
        spill_dir = tempfile.mkdtemp(prefix=".spill-", dir=graph_dir)
        paths = [os.path.join(spill_dir, f"part{r}.bin") for r in range(n_parts)]
        spills = [open(p, "wb") for p in paths]
        try:
            in_cnt, out_cnt = _spill_edges(pf, new_id, ranges, spills, dev, chunk)
        finally:
            for f in spills:
                f.close()
        del new_id
        order = order.cpu()
        cfg = _head(args, ranges, 0)
        for r in range(n_parts):
            cfg[f"part-{r}"] = _streamed_part(pf, r, ranges, order, in_cnt, out_cnt, paths[r],
                                              os.path.join(graph_dir, f"part{r}"), dev)
            os.remove(paths[r])
        cfg["num_edges"] = sum(cfg[f"part-{r}"]["n_edges"] for r in range(n_parts))
        del order, in_cnt, out_cnt
        _stream_features(pf, part, [cfg[f"part-{r}"]["n_in"] for r in range(n_parts)], graph_dir, chunk)
        _finish(graph_dir, part_config, cfg, (pf.n_feat, pf.n_class, int(pf.train.sum())))
        return part_config
    except BaseException:
        if created:
            shutil.rmtree(graph_dir, ignore_errors=True)
        else:                                              # a store directory without a config holds no complete part
            for r in range(args.n_partitions):
                shutil.rmtree(os.path.join(graph_dir, f"part{r}"), ignore_errors=True)
        raise
    finally:
        if spill_dir is not None:
            shutil.rmtree(spill_dir, ignore_errors=True)


def _load_array(path: str, mmap: bool) -> torch.Tensor:
    a = np.load(path, mmap_mode='r' if mmap else None, allow_pickle=False)
    return torch.from_numpy(np.array(a))        # a private, writable copy (the mapping itself is read-only)


def _read_part(graph_dir: str, part_config: str, cfg: dict, rank: int, device, mmap: bool):
    """``(subg, node_dict, gpb)`` of part ``rank`` of the (checked) part config ``cfg``, read from ``part_config``."""
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
    return subg, node_dict, gpb


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
    subg, node_dict, gpb = _read_part(graph_dir, part_config, cfg, rank, device, mmap)
    with open(os.path.join(graph_dir, 'meta.json')) as f:
        meta = json.load(f)
    args.n_feat, args.n_class, args.n_train = meta['n_feat'], meta['n_class'], meta['n_train']   # utils.py:134-138
    return subg, node_dict, gpb


def load_eval_partition(args, which: str, rank: int, device: Optional[torch.device] = None, mmap: bool = True):
    """``(subg, node_dict, gpb)`` of part ``rank`` of the evaluation set ``which`` (``'val'`` | ``'test'``), the
    contract of ``load_partition``; ``node_dict`` holds ``which + '_mask'`` and the degrees of that graph."""
    eval_dir, eval_config = _eval_dirs(args, which)
    if not os.path.exists(eval_config):
        raise FileNotFoundError(f"{eval_config}: no such evaluation partition config; run graph_partition(args) with "
                                "--eval --parallel-eval --inductive first (main.py does unless --skip-partition)")
    with open(eval_config) as f:
        cfg = json.load(f)
    if cfg.get("format_version") != FORMAT_VERSION:
        raise RuntimeError(f"{eval_config}: format version {cfg.get('format_version')} != {FORMAT_VERSION}")
    _check_eval(cfg, args, which, eval_config)
    if not 0 <= rank < cfg["num_parts"]:
        raise IndexError(f"part {rank} of {cfg['num_parts']}")
    return _read_part(eval_dir, eval_config, cfg, rank, device, mmap)


def load_as_partition(args, rank: int, device: Optional[torch.device] = None) -> Partition:
    """The same part wrapped as the in-memory ``Partition`` record the tests and tools pass around."""
    subg, nd, gpb = load_partition(args, rank, device)
    return Partition(rank, gpb.num_partitions(), subg, nd, gpb,
                     {"n_feat": args.n_feat, "n_class": args.n_class, "n_train": args.n_train})
