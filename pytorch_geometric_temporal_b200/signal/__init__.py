from .data import Data  # noqa: F401
from .static_graph_temporal_signal import StaticGraphTemporalSignal  # noqa: F401
from .static_graph_temporal_signal_batch import StaticGraphTemporalSignalBatch  # noqa: F401
from .dynamic_graph_signal import (DynamicGraphTemporalSignal, DynamicGraphStaticSignal,  # noqa: F401
                                   DynamicGraphTemporalSignalBatch, DynamicGraphStaticSignalBatch)
from .train_test_split import temporal_signal_split  # noqa: F401
from .index_dataset import IndexDataset, IndexBatchLoader, DevicePrefetcher, shard_indices, index_splits  # noqa: F401
from .static_hetero_graph_temporal_signal import StaticHeteroGraphTemporalSignal, HeteroData  # noqa: F401
