"""Launched by torchrun on 2 GPUs (tests/test_gpu_gat.py): the data-parallel replica check of
tests/dist_replica_check.py with the GAT encoder (4 heads, Set2Set 2 iterations x 2 LSTM layers) in place of GIN:
after 5 steps parameters, EMA parameters, queue and queue pointer hash identically on both ranks, and the first
step's summed gradient equals the sum of the two single-GPU shards."""
import dist_replica_check as drc

import gcc_b200.models as models

_GraphEncoder = models.GraphEncoder


def _gat_encoder(**kw):
    kw.update(gnn_model="gat", num_heads=4, num_step_set2set=2, num_layer_set2set=2)
    return _GraphEncoder(**kw)


models.GraphEncoder = _gat_encoder      # dist_replica_check.build imports it from gcc_b200.models at call time

if __name__ == "__main__":
    drc.main()
