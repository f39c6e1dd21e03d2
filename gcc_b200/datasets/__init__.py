from . import synthetic  # noqa: F401


def __getattr__(name):          # lazy: graph_dataset pulls in torch + the CUDA library
    if name in ("LoadBalanceGraphDataset", "NodeClassificationDataset", "GraphClassificationDataset", "DeviceGraph",
                "BatchBuffers"):
        from . import graph_dataset
        return getattr(graph_dataset, name)
    if name in ("BatchedSubgraphs", "batcher"):
        from . import data_util
        return getattr(data_util, name)
    raise AttributeError(name)
