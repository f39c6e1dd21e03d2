"""CPU: GraphEncoder(gnn_model="gat") as a module -- the reference's state_dict keys and shapes, the parameter count,
initial weights under torch.manual_seed against a plain-torch construction in the reference's order, and the
drivers' option parsing."""
import pytest
import torch

import gat_oracle
from gcc_b200.models import GraphEncoder
from gcc_b200.models import layout as glayout


def _enc(L, nh, H=64, K=3, P=32, D=16, maxdeg=512):
    return GraphEncoder(positional_embedding_size=P, max_degree=maxdeg, degree_embedding_size=D, output_dim=H,
                        node_hidden_dim=H, num_layers=L, num_heads=nh, num_step_set2set=6, num_layer_set2set=K,
                        norm=True, gnn_model="gat", degree_input=True)


@pytest.mark.parametrize("L,nh", [(2, 1), (2, 4), (5, 1), (5, 4)])
def test_state_dict_keys_shapes_and_count(L, nh):
    H, K, din = 64, 3, 49
    m = _enc(L, nh)
    want = {}
    for i in range(L):
        want["gnn.layers.%d.gnn.fc.weight" % i] = (H, din if i == 0 else H)
        want["gnn.layers.%d.gnn.attn_l" % i] = (1, nh, H // nh)
        want["gnn.layers.%d.gnn.attn_r" % i] = (1, nh, H // nh)
    want["degree_embedding.weight"] = (513, 16)
    for k in range(K):
        want["set2set.lstm.weight_ih_l%d" % k] = (4 * H, 2 * H if k == 0 else H)
        want["set2set.lstm.weight_hh_l%d" % k] = (4 * H, H)
        want["set2set.lstm.bias_ih_l%d" % k] = (4 * H,)
        want["set2set.lstm.bias_hh_l%d" % k] = (4 * H,)
    want["lin_readout.0.weight"], want["lin_readout.0.bias"] = (H, 2 * H), (H,)
    want["lin_readout.2.weight"], want["lin_readout.2.bias"] = (H, H), (H,)
    sd = m.state_dict()
    assert {k: tuple(v.shape) for k, v in sd.items()} == want        # no buffers
    n = sum(p.numel() for p in m.parameters())
    assert n == m.n_live == m.flat_params.numel() == sum(torch.Size(s).numel() for s in want.values())
    # every parameter is a view of the one flat buffer
    for p in m.parameters():
        assert p.data_ptr() >= m.flat_params.data_ptr()
        assert p.data_ptr() + 4 * p.numel() <= m.flat_params.data_ptr() + 4 * m.flat_params.numel()


@pytest.mark.parametrize("L,nh", [(2, 4), (5, 1)])
def test_initial_weights_follow_the_reference_construction_order(L, nh):
    torch.manual_seed(123)
    m = _enc(L, nh)
    torch.manual_seed(123)
    ref = gat_oracle.reference_init(L, 64, nh, 49, 512, 16, 3)
    sd = m.state_dict()
    assert set(ref) == set(sd)
    for k, v in ref.items():
        assert torch.equal(sd[k], v.reshape(sd[k].shape)), k


def test_load_state_dict_round_trip_and_hidden_multiple_of_heads():
    a, b = _enc(2, 4), _enc(2, 4)
    b.load_state_dict(a.state_dict())
    assert torch.equal(a.flat_params, b.flat_params)
    with pytest.raises(ValueError):
        _enc(2, 3, H=64)


def test_layout_mirror_matches_module():
    m = _enc(3, 4, K=2)
    sl, total = glayout.gat_param_slices(m.cfg)
    assert total == m.n_live
    sd = m.state_dict()
    for k, (off, shape) in sl.items():
        assert torch.equal(m.flat_params[off:off + torch.Size(shape).numel()].view(shape), sd[k])


def test_mpnn_stays_refused_with_the_reason():
    with pytest.raises(NotImplementedError, match="graph_encoder.py:188"):
        GraphEncoder(gnn_model="mpnn", degree_input=True)


def test_train_parses_model_gat():
    import train
    args = train.parse_option(["--model", "gat"])
    assert args.model == "gat"
    with pytest.raises(SystemExit):
        train.parse_option(["--model", "mpnn"])
