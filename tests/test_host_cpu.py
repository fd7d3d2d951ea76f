"""CPU tests of the product's host side: the C-ABI library loads and exports every symbol include/bnsgcn.h
declares (no compute calls without a GPU), the partition contract, and the exchange metadata
(get_boundary / get_pos / send-recv sizes / data_transfer) under torch.distributed gloo with world_size 2."""
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_exports_every_declared_symbol(built):
    from bns_gcn_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "bnsgcn.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(bns_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    for name in declared:
        assert hasattr(_lib.lib, name)
    assert _lib.lib.bns_abi_version() == _lib.ABI_VERSION
    assert _lib.lib.bns_spmm_workspace_bytes(None, 16) == 0
    assert _lib.lib.bns_launch_count() >= 0


def test_product_refuses_cpu_tensors(built):
    """No CPU fallback: the ops fail loudly on non-CUDA inputs."""
    from bns_gcn_b200 import _lib, ops
    with pytest.raises(_lib.BnsError):
        ops.DeviceGraph.from_csr(torch.zeros(2, dtype=torch.int64), torch.zeros(0, dtype=torch.int32), 1)
    with pytest.raises(_lib.BnsError):
        ops.gather_div(torch.zeros(2, 4), torch.zeros(1, dtype=torch.int64), 1.0)


def test_missing_library_fails_loudly(tmp_path):
    code = ("import sys; sys.path.insert(0, %r); import bns_gcn_b200._lib as L\n" % ROOT)
    import subprocess
    env = dict(os.environ)
    src = os.path.join(ROOT, "bns-gcn_b200", "csrc", "libbnsgcn.so")
    bak = src + ".bak_test"
    if not os.path.exists(src):
        pytest.skip("library not built")
    os.rename(src, bak)
    try:
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env)
    finally:
        os.rename(bak, src)
    assert r.returncode != 0 and "no CPU fallback" in r.stderr.replace("\n", " ")


@pytest.mark.parametrize("method", ["random", "metis"])
def test_partition_contract(method):
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200.data import make_graph, partition_graph
    fg = make_graph("small", seed=1, device=torch.device("cpu"))
    # generator contract: one self loop per node, no multi-edges, symmetric
    dst = fg.dst()
    key = dst * fg.n_nodes + fg.src
    assert key.unique().numel() == key.numel()
    assert int((dst == fg.src).sum()) == fg.n_nodes
    assert torch.equal(torch.sort(fg.src * fg.n_nodes + dst)[0], torch.sort(key)[0])
    P = 4
    parts = partition_graph(fg, P, method, seed=1, device=torch.device("cpu"))
    ranges = parts[0].gpb.ranges
    assert int(ranges[-1]) == fg.n_nodes and torch.all(ranges[1:] - ranges[:-1] > 0)
    n_edges = 0
    for r, p in enumerate(parts):
        nd, g = p.node_dict, p.graph
        assert g.n_in == int(ranges[r + 1] - ranges[r])
        assert torch.equal(nd["_ID"][:g.n_in], torch.arange(int(ranges[r]), int(ranges[r + 1])))     # contiguous
        assert nd["inner_node"][:g.n_in].all() and not nd["inner_node"][g.n_in:].any()
        assert torch.all(nd["part_id"][:g.n_in] == r) and torch.all(nd["part_id"][g.n_in:] != r)
        assert torch.equal(g.indptr[1:] - g.indptr[:-1], nd["in_deg"])          # ALL in-edges of inner nodes, full degree
        assert g.indices.max() < g.n_in + g.n_halo and g.indices[g.indices >= g.n_in].unique().numel() == g.n_halo
        n_edges += g.num_edges()
        assert p.meta["n_train"] == int(fg.train_mask.sum())
    assert n_edges == fg.n_edges


def _gloo_worker(rank, world, port, out_dir, use_store=False):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_graph, partition_graph
    from bns_gcn_b200.helper import context as ctx
    from bns_gcn_b200.helper.utils import TransferTag, data_transfer, get_boundary
    fg = make_graph("tiny", seed=0, device=torch.device("cpu"))
    if use_store:
        # main.py's flow under torchrun: rank 0 writes the partition store, everybody loads its own part from disk
        import argparse
        from bns_gcn_b200.data import graph_partition, load_as_partition
        a = argparse.Namespace(dataset="tiny", n_partitions=world, partition_method="random", partition_obj="vol",
                               inductive=False, part_path=os.path.join(out_dir, "partition"), graph_name="")
        if rank == 0:
            graph_partition(a, fg=fg, device=torch.device("cpu"))
        dist.barrier()
        p = load_as_partition(a, rank)
        assert (a.n_feat, a.n_class, a.n_train) == (fg.n_feat, fg.n_class, int(fg.train_mask.sum()))
    else:
        p = partition_graph(fg, world, "random", seed=0, device=torch.device("cpu"))[rank]
    assert ctx.comm().kind == "dist" and ctx.comm().backend == "gloo"
    boundary = get_boundary(p.node_dict, p.gpb)
    pos = train.get_pos(p.node_dict, p.gpb)
    send_size, ratio = train.get_send_size(boundary, 0.5)
    recv_size = train.get_recv_size(p.node_dict, 0.5)
    out_deg = train.collect_out_degree(p.node_dict, boundary)
    sel = [None if b is None else b[torch.randperm(b.numel(), generator=torch.Generator().manual_seed(rank))[:s]]
           for b, s in zip(boundary, send_size)]
    hops = data_transfer(sel, [torch.Size([s]) for s in recv_size], tag=TransferTag.NODE, dtype=torch.long)
    torch.save({"boundary": boundary, "pos": pos, "send": send_size, "ratio": ratio, "recv": recv_size,
                "out_deg": out_deg, "sel": sel, "hops": hops, "nid": p.node_dict["_ID"], "n_in": p.graph.n_in,
                "ranges": p.gpb.ranges, "global_out_deg": fg.out_degrees()}, os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world,use_store", [(2, False), (2, True), (4, False)])
def test_exchange_metadata_gloo(tmp_path, world, use_store):
    """get_boundary / get_pos / send-recv sizes / data_transfer over torch.distributed gloo, ``world`` processes."""
    import torch.multiprocessing as mp
    mp.spawn(_gloo_worker, args=(world, 29650 + 2 * world + int(use_store), str(tmp_path), use_store), nprocs=world, join=True)
    r = [torch.load(os.path.join(tmp_path, f"r{i}.pt")) for i in range(world)]
    gold = torch.load(os.path.join(ROOT, "tests", "golden", "ref_graphsage_p2.pt"))["ranks"] if world == 2 else None
    for me in range(world):
        for other in range(world):
            if other == me:
                continue
            a, b = r[me], r[other]
            if gold is not None:
                assert torch.equal(a["boundary"][other], gold[me]["boundary"][other])     # == the reference's get_boundary
            assert a["send"][other] == b["recv"][me] == int(0.5 * a["boundary"][other].numel())
            assert abs(a["ratio"][other] - a["send"][other] / a["boundary"][other].numel()) < 1e-12
            assert torch.equal(b["hops"][me], a["sel"][other])                            # exchange exactness
            # pos maps the sender's local ids onto my halo slots: the global ids agree
            mine = b["pos"][me][a["sel"][other]]
            assert torch.all(mine >= b["n_in"])
            assert torch.equal(b["nid"][mine], a["sel"][other] + int(a["ranges"][me]))
        # merged out-degree vector covers [inner | halo]
        assert r[me]["out_deg"].numel() == r[me]["nid"].numel()


def _local_generator_worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200 import train
    from bns_gcn_b200.data import make_local_partition
    from bns_gcn_b200.helper.utils import get_boundary
    p = make_local_partition("papers100m", rank, world, seed=0, device=torch.device("cpu"), scale=0.0002)
    boundary = get_boundary(p.node_dict, p.gpb)
    send_size, _ = train.get_send_size(boundary, 0.1)
    recv_size = train.get_recv_size(p.node_dict, 0.1)
    out_deg = train.collect_out_degree(p.node_dict, boundary)
    ip, ix = p.graph.indptr, p.graph.indices
    torch.save({"boundary": boundary, "send": send_size, "recv": recv_size, "nid": p.node_dict["_ID"], "n_in": p.graph.n_in,
                "n_halo": p.graph.n_halo, "ranges": p.gpb.ranges, "part_id": p.node_dict["part_id"], "indptr": ip,
                "indices": ix, "in_deg": p.node_dict["in_deg"], "out_deg_all": out_deg, "meta": p.meta},
               os.path.join(out_dir, f"r{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


def test_per_rank_generator_partitions_agree_gloo(tmp_path):
    """data.make_local_partition (the papers100M-shape path: every rank generates its own piece, the graph never exists
    as a whole): the pieces of 2 ranks form ONE consistent partitioned graph -- contiguous ownership, halo ids owned by
    the peer and sorted, boundary lists that mirror the peer's halo, matching send / receive sizes, exact in-degrees,
    one self loop per node, no duplicate entries."""
    import torch.multiprocessing as mp
    world = 2
    mp.spawn(_local_generator_worker, args=(world, 29671, str(tmp_path)), nprocs=world, join=True)
    r = [torch.load(os.path.join(tmp_path, f"r{i}.pt")) for i in range(world)]
    assert torch.equal(r[0]["ranges"], r[1]["ranges"]) and r[0]["meta"] == r[1]["meta"]
    for me in range(world):
        a, other = r[me], 1 - me
        b = r[other]
        n_in, lo, hi = a["n_in"], int(a["ranges"][me]), int(a["ranges"][me + 1])
        assert n_in == hi - lo and torch.equal(a["nid"][:n_in], torch.arange(lo, hi))
        halo = a["nid"][n_in:]
        assert halo.numel() == a["n_halo"] and torch.all(halo[1:] > halo[:-1])             # sorted, unique
        assert torch.all((halo < lo) | (halo >= hi)) and torch.all(a["part_id"][n_in:] == other)
        # what the peer may be asked to send me is exactly my halo, in the peer's local numbering
        assert torch.equal(b["boundary"][me] + int(a["ranges"][other]), halo)
        assert a["recv"][other] == b["send"][me] == int(0.1 * halo.numel())
        ip, ix = a["indptr"], a["indices"].long()
        assert torch.equal(ip[1:] - ip[:-1], a["in_deg"]) and int(ip[-1]) == ix.numel()
        rows = torch.repeat_interleave(torch.arange(n_in), ip[1:] - ip[:-1])
        key = rows * (n_in + a["n_halo"]) + ix
        assert key.unique().numel() == key.numel()                                          # no duplicate entries
        assert int(((ix == rows).long()).sum()) == n_in                                     # one self loop per node
        assert torch.unique(ix[ix >= n_in]).numel() == a["n_halo"]                          # every halo node is used
        assert a["out_deg_all"].numel() == n_in + a["n_halo"]


def test_dense_split_k_plan_is_sane_without_a_gpu(built):
    """``bns_dense_nt_workspace_bytes`` is pure host arithmetic (SM count falls back to 132, the H100 SXM's, without a device): the
    weight-gradient contraction is cut into slices of at most 48 k-blocks of 32 rows (accumulation-chain bound,
    csrc/dense_tc.cuh), never more slices than k-blocks, and no workspace when one slice suffices."""
    from bns_gcn_b200 import _lib
    f = _lib.lib.bns_dense_nt_workspace_bytes
    assert f(32, 128, 128) == 0 and f(0, 128, 128) == 0 and f(100, 0, 8) == 0
    for R, n1, n2 in [(232965, 256, 1204), (232965, 256, 256), (58242, 256, 1204), (29121, 44, 256), (1000, 136, 100)]:
        b = f(R, n1, n2)
        assert b % (n1 * n2 * 4) == 0
        splits = b // (n1 * n2 * 4) if b else 1
        kb = (R + 31) // 32
        assert 1 <= splits <= kb
        assert (kb + splits - 1) // splits <= 48 + 5, (R, n1, n2, splits)      # <= 48 up to the -10 % wave rounding
    # contractions of more than 1,024 x 48 k-blocks (the papers100M per-rank rows): never above 48 k-blocks per slice
    for R, n1, n2 in [(111_059_956 // 8, 256, 256), (111_059_956 // 8, 44, 256), (2_000_000, 256, 1204)]:
        kb = (R + 31) // 32
        splits = f(R, n1, n2) // (n1 * n2 * 4)
        assert splits >= (kb + 47) // 48 > 1024, (R, n1, n2, splits)
    assert _lib.lib.bns_colsum_workspace_bytes(256) == 132 * 4 * 64 * 16


def _planted_partition_graph(n, P, deg_in, deg_out, seed=0):
    """Symmetric stochastic-block-model graph with one self loop per node (the generator's contract) and its blocks."""
    from bns_gcn_b200.data import FullGraph
    g = torch.Generator().manual_seed(seed)
    blk = torch.randint(0, P, (n,), generator=g)
    order = torch.argsort(blk)
    starts, sizes = torch.searchsorted(blk[order], torch.arange(P)), torch.bincount(blk, minlength=P)
    m_in, m_out = n * deg_in // 2, n * deg_out // 2
    u = torch.randint(0, n, (m_in,), generator=g)
    v = order[starts[blk[u]] + (torch.rand(m_in, generator=g) * sizes[blk[u]]).long().clamp(max=sizes[blk[u]] - 1)]
    a = torch.cat([u, torch.randint(0, n, (m_out,), generator=g)])
    b = torch.cat([v, torch.randint(0, n, (m_out,), generator=g)])
    keep = a != b
    lo, hi = torch.minimum(a[keep], b[keep]), torch.maximum(a[keep], b[keep])
    key = torch.unique(lo * n + hi)
    lo, hi, loops = key // n, key % n, torch.arange(n)
    dst, src = torch.cat([lo, hi, loops]), torch.cat([hi, lo, loops])
    o = torch.argsort(dst * n + src)
    dst, src = dst[o], src[o]
    indptr = torch.zeros(n + 1, dtype=torch.int64)
    indptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n), 0)
    z = torch.zeros(n, dtype=torch.bool)
    return FullGraph(n, indptr, src, torch.zeros(n, 1), torch.zeros(n, dtype=torch.int64), z, z, z, 2), blk


@pytest.mark.parametrize("objective", ["cut", "vol"])
def test_metis_standin_finds_planted_structure(objective):
    """``--partition-method metis`` (RCM blocks + balanced label propagation on ``--partition-obj``): on a graph with
    4 planted communities it must land near the planted cut -- far below what ``random`` gives -- within the size cap,
    and the refinement must never return something worse than it was given."""
    import bns_gcn_b200  # noqa: F401
    from bns_gcn_b200.data import assign_parts, partition_quality, refine_label_propagation
    fg, blk = _planted_partition_graph(8000, 4, 16, 2)
    planted = partition_quality(fg, blk, 4)
    rnd = partition_quality(fg, assign_parts(fg, 4, "random", 0), 4)
    part = assign_parts(fg, 4, "metis", 0, objective)
    q = partition_quality(fg, part, 4)
    assert q[objective] <= 1.5 * planted[objective] and q[objective] < 0.5 * rnd[objective], (q, planted, rnd)
    assert q["max_size"] <= int(1.03 * 8000 / 4) + 1 and q["min_size"] >= int(0.97 * 8000 / 4)
    # monotone: refining a random assignment never makes it worse
    start = assign_parts(fg, 4, "random", 1)
    better = refine_label_propagation(fg, start, 4, objective)
    assert partition_quality(fg, better, 4)[objective] <= partition_quality(fg, start, 4)[objective]


def test_integration_md_examples_have_the_abi_arity(built):
    """Every `_L.bns_*(...)` call shown in INTEGRATION.md passes as many arguments as include/bnsgcn.h declares (the
    reference-side stubs a maintainer would paste must at least bind)."""
    from bns_gcn_b200 import _lib
    txt = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    seen = 0
    for m in re.finditer(r"_L\.(bns_[a-z0-9_]+)\(", txt):
        name, i, depth, commas = m.group(1), m.end(), 1, 0
        while depth > 0 and i < len(txt):
            ch = txt[i]
            if ch in "([{":
                depth += 1
            elif ch in ")]}":
                depth -= 1
            elif ch == "," and depth == 1:
                commas += 1
            i += 1
        body = txt[m.end():i - 1].strip()
        n_args = 0 if not body else commas + 1
        assert name in _lib.SIGNATURES, name
        assert n_args == len(_lib.SIGNATURES[name][1]), (name, n_args, len(_lib.SIGNATURES[name][1]))
        seen += 1
    assert seen >= 30


def test_header_is_plain_c_and_links(built, tmp_path):
    """include/bnsgcn.h is the drop-in boundary: a C (not C++) translation unit that includes nothing but that header
    compiles with -Wall -Werror -pedantic, links against libbnsgcn.so and can call the entry points that need no GPU."""
    import shutil
    import subprocess
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    src = tmp_path / "abi_probe.c"
    src.write_text(
        '#include "bnsgcn.h"\n'
        '#include <stdio.h>\n'
        '#include <string.h>\n'
        'int main(void) {\n'
        '    struct bns_epoch_maps m; struct bns_put_all p; struct bns_derive_entry d;\n'
        '    memset(&m, 0, sizeof m); memset(&p, 0, sizeof p); memset(&d, 0, sizeof d);\n'
        '    if (bns_abi_version() != BNS_ABI_VERSION) return 2;\n'
        '    if (bns_spmm_workspace_bytes(NULL, 16) != 0) return 3;\n'
        '    if (bns_spmm_sum_f32(NULL, NULL, 0, 0, NULL, 0, NULL, NULL, NULL, NULL, NULL, 0, 0, 0, 0, NULL, 0, NULL) >= 0) return 4;\n'
        '    if (strlen(bns_last_error()) == 0) return 5;\n'
        '    printf("abi %d peers %d\\n", bns_abi_version(), BNS_MAX_PEERS);\n'
        '    return 0;\n'
        '}\n')
    lib_dir = os.path.join(ROOT, "bns-gcn_b200", "csrc")
    exe = tmp_path / "abi_probe"
    cc = subprocess.run(["gcc", "-std=c11", "-Wall", "-Werror", "-pedantic", "-I", os.path.join(ROOT, "include"), str(src),
                         "-o", str(exe), "-L", lib_dir, "-lbnsgcn", f"-Wl,-rpath,{lib_dir}"],
                        capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True)
    assert run.returncode == 0, (run.returncode, run.stdout, run.stderr)
    assert run.stdout.startswith("abi ")
