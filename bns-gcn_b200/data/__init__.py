from .synthetic import FullGraph, SHAPES, make_graph, make_local_partition
from .partition import (NID, GraphPartitionBook, LocalGraph, Partition, partition_graph, extract_partition,
                        assign_parts, relabel, induced_subgraph, refine_label_propagation, partition_quality)
from .files import DATA_SOURCES, DataFileError, data_source, load_files, load_graph, read_papers100m
from .store import (graph_partition, load_partition, load_as_partition, save_partition, default_graph_name,
                    eval_partitions, load_eval_partition, papers100m_partition, check_papers100m)
