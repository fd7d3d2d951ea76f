"""Command-line flags.  The reference's flag set (helper/parser.py:4-61) is an interface, so names, spellings
(``--a-b`` and ``--a_b``), types and defaults are kept; it is declared as a table here, followed by the flags that
only exist in this build."""
import argparse

# (flag, type or None for a switch, default, extra argparse keywords)
_REFERENCE_FLAGS = [
    ("dataset", str, "reddit", dict(help="synthetic shape to generate: reddit | ogbn-products | yelp | "
                                         "ogbn-papers100m | synthetic-10k | small | tiny; with --data-source files, the "
                                         "dataset to read: reddit | ogbn-products | yelp | ogbn-papers100m.  "
                                         "ogbn-papers100m (also papers100m) is partitioned by streaming, one part at a "
                                         "time: only with --partition-method random, --partition-balance nodes, "
                                         "transductive, and --parallel-eval or --no-eval")),
    ("data-path", str, "./dataset/", {}),
    ("part-path", str, "./partition/", {}),
    ("graph-name", str, "", {}),
    ("model", str, "graphsage", dict(help="graphsage | gcn | gat | gatv2 | graphsage-pool | transformer.  gatv2 (NEW) is GAT with "
                                          "dynamic attention (GATv2Conv: the score attn . leaky_relu(z_src[u] + z_dst[v]) "
                                          "per head), on the same layer stack, heads, norms and limits as gat.  "
                                          "graphsage-pool (NEW) is GraphSAGE with the max-pooling aggregator (SAGEConv "
                                          "'pool': a max over the sampled neighbours of relu(fc_pool(h)), exchanged rows "
                                          "unscaled); --heads is ignored.  transformer (NEW) is the graph transformer "
                                          "layer (TransformerConv: scaled dot-product attention <q_v, k_u> / sqrt(C), "
                                          "heads averaged, plus a root weight), on GAT's stack, heads, norms and "
                                          "limits, exchanged rows unscaled")),
    ("dropout", float, 0.5, {}),
    ("lr", float, 1e-2, {}),
    ("sampling-rate", float, 1, {}),
    ("heads", int, 1, {}),
    ("n-epochs", int, 200, {}),
    ("n-partitions", int, 2, {}),
    ("n-hidden", int, 16, {}),
    ("n-layers", int, 2, {}),
    ("log-every", int, 10, {}),
    ("weight-decay", float, 0, {}),
    ("norm", None, "layer", dict(choices=["layer", "batch"])),
    ("partition-obj", None, "vol", dict(choices=["vol", "cut"])),
    ("partition-method", None, "metis", dict(choices=["metis", "random", "multilevel"],
                                             help="metis: the stand-in (reverse Cuthill-McKee blocks refined by balanced "
                                                  "label propagation, on the host or the given device); random; "
                                                  "NEW multilevel: a multilevel k-way partitioner on the GPU (coarsen, "
                                                  "initial partition, refine on --partition-obj), 2 to 64 parts")),
    ("n-linear", int, 0, {}),
    ("use-pp", "switch", False, {}),
    ("inductive", "switch", False, {}),
    ("fix-seed", "switch", False, {}),
    ("seed", int, 0, {}),
    ("backend", str, "nccl", dict(help="exchange transport: nccl (staged all-to-all) | p2p (peer-mapped slabs over "
                                       "NVLink); the reference's gloo / mpi host-staged transports are what this "
                                       "replaces")),
    ("port", int, 18118, {}),
    ("master-addr", str, "127.0.0.1", {}),
    ("node-rank", int, 0, {}),
    ("parts-per-node", int, 10, {}),
]


def _spellings(flag: str):
    dashed = "--" + flag
    return (dashed,) if "-" not in flag else (dashed, dashed.replace("-", "_").replace("__", "--", 1))


def build_parser():
    parser = argparse.ArgumentParser(description='BNS-GCN (H100-native hot path)')
    for flag, kind, default, extra in _REFERENCE_FLAGS:
        if kind == "switch":
            parser.add_argument(*_spellings(flag), action='store_true')
        elif kind is None:
            parser.add_argument(*_spellings(flag), default=default, **extra)
        else:
            parser.add_argument(*_spellings(flag), type=kind, default=default, **extra)
    parser.add_argument('--skip-partition', action='store_true')
    # --eval / --no-eval write the same destination; evaluation is on unless --no-eval is given (parser.py:57-59)
    parser.add_argument('--eval', action='store_true')
    parser.add_argument('--no-eval', action='store_false', dest='eval')
    parser.set_defaults(eval=True)
    # only here
    parser.add_argument(*_spellings("sampler-seed"), type=int, default=0,
                        help="NEW: Philox seed of the boundary sampler (the reference draws from unseeded numpy)")
    parser.add_argument(*_spellings("parallel-eval"), action='store_true',
                        help="NEW: with --eval, every rank evaluates its own nodes on its partition (the whole halo "
                             "exchanged layer by layer) instead of rank 0 evaluating the full graph alone; the full "
                             "graph is never built.  With --inductive, on partitions of the train | val subgraph "
                             "and of the full graph, which the partition step writes beside the training parts")
    parser.add_argument(*_spellings("data-source"), default="synthetic", choices=["synthetic", "files"],
                        help="NEW: where the graph comes from.  synthetic generates the --dataset shape from a seed.  "
                             "files reads reddit, yelp, ogbn-products or ogbn-papers100m from the files DGL / OGB "
                             "leave under --data-path (reddit/, yelp/, ogbn_products/ and ogbn_papers100M/ raw and "
                             "split/); the store's default graph name then carries a 'files' token")
    parser.add_argument(*_spellings("agg-dtype"), default="f32", choices=["f32", "bf16", "fp8"],
                        help="NEW: element type of the rows the wide (hidden-width) aggregation passes gather.  bf16 "
                             "rounds them to bf16 (nearest even) before each pass -- h_u forward, the transposed "
                             "passes' input gradient backward -- and sums in f32: half the gathered bytes, and results "
                             "that no longer match the reference to 1e-4.  fp8 stores the same rows as e4m3 (nearest "
                             "even) with one power-of-two scale per row: a quarter of the f32 bytes; hidden widths "
                             "must be multiples of 16.  Only with the fused training step (GraphSAGE / GCN, --use-pp, "
                             "--norm layer, no --n-linear)")
    parser.add_argument(*_spellings("comm-dtype"), default="f32", choices=["f32", "bf16", "fp8"],
                        help="NEW: element type of the boundary rows the training exchange moves.  bf16 rounds each "
                             "sampled row H[selected]/ratio, and each returned halo gradient row, to bf16 (nearest even) "
                             "at the sender: half the wire and slab bytes; the receiver widens and sums in f32.  fp8 "
                             "sends each such row as e4m3 codes plus one power-of-two scale (the --agg-dtype fp8 row "
                             "format): F + 4 bytes a row; the hidden width must be a multiple of 16.  Only with the "
                             "fused training step (GraphSAGE / GCN, --use-pp, --norm layer, no --n-linear)")
    parser.add_argument(*_spellings("dense-dtype"), default="f32", choices=["f32", "bf16", "fp8"],
                        help="NEW: operand precision of the training step's dense layers.  f32 runs the f32-accurate "
                             "3xTF32 tensor-core scheme; bf16 rounds every GEMM operand to bf16 (nearest even) inside "
                             "the kernel and sums in f32: one bf16 tensor-core product instead of three TF32 ones, and "
                             "results that no longer match the reference to 1e-4.  fp8 feeds the forward and "
                             "input-gradient GEMMs with fp8 rows of both operands (e4m3 codes plus one power-of-two "
                             "scale per row, the --agg-dtype fp8 format; sums promoted to f32 every 128 products); the "
                             "weight gradients run the bf16 products, because their contraction runs over the nodes, "
                             "where a per-row scale does not factor out.  Master weights, gradients, the all-reduce, "
                             "Adam, the loss and evaluation stay f32.  Only with the fused training step (GraphSAGE / "
                             "GCN, --use-pp, --norm layer, no --n-linear)")
    parser.add_argument(*_spellings("partition-balance"), default="nodes", choices=["nodes", "edges"],
                        help="NEW: what every --partition-method balances.  nodes: each part's node count within 3 %% "
                             "of N / P.  edges: that, and each part's in-edges (the edges whose destination it owns, "
                             "loops included: a rank's aggregation work) at most int(1.03 E / P) plus the largest "
                             "in-degree; a method that cannot meet a bound raises.  The store's default graph name "
                             "then carries an 'edges' token")
    parser.add_argument(*_spellings("save-state-every"), type=int, default=0,
                        help="NEW: after every N-th epoch, and after the last one, all ranks write the training state "
                             "(weights, Adam moments and step, the CUDA generators, the evaluator's best model, the "
                             "seed) to checkpoint/<graph_name>_state/, which --resume continues from.  0: never.  "
                             "Independent of --eval")
    parser.add_argument(*_spellings("resume"), action='store_true',
                        help="NEW: before the first epoch, load the state saved under this run's graph name and "
                             "continue with the next epoch up to --n-epochs (which counts all epochs).  The resumed run "
                             "is bit-identical to an uninterrupted one")
    parser.add_argument(*_spellings("cuda-graph"), action='store_true',
                        help="NEW: after this process's first three epochs, which run eagerly, capture one epoch into a "
                             "CUDA graph and run every later epoch as one replay of it: the same losses and weights, "
                             "bit for bit, without the host enqueueing each epoch's launches.  Comm(s) / Reduce(s) are "
                             "timed inside the replay by GPU clock stamps.  Refused (before any setup) for ranks that "
                             "are threads of one process and for the staged --backend nccl at more than 2 partitions")
    return parser


def create_parser(argv=None):
    return build_parser().parse_args(argv)
