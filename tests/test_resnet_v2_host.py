"""Keras ResNet50V2 / ResNet101V2 / ResNet152V2 (keras_applications 1.0.8 ``resnet_common.py``) on the CPU: the graph,
the layer names, the synthetic-weight rule, partitions, and one pre-activation block restated with torch.nn.functional."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from defer_b200 import applications, dag_util
from defer_b200 import keras_like as K
from oracle import keras_ref, torch_cpu

V2 = {"ResNet50V2": (25_613_800, 16), "ResNet101V2": (44_675_560, 33), "ResNet152V2": (60_380_648, 50)}


@pytest.fixture(scope="module")
def models():
    return {name: getattr(applications, name)() for name in V2}


@pytest.mark.parametrize("name", list(V2))
def test_parameter_counts_and_residual_adds(models, name):
    m = models[name]
    params, n_adds = V2[name]
    assert m.count_params() == params
    adds = applications.residual_add_names(m)
    assert len(adds) == n_adds
    assert all(a.endswith("_out") for a in adds)
    assert adds[0] == "conv2_block1_out" and adds[-1] == "conv5_block3_out"
    assert len(applications.default_cuts(m, 4)) == 3


def test_layer_names_and_structure(models):
    m = models["ResNet50V2"]
    names = [l.name for l, _ in m.iter_nodes()]
    assert names[1:5] == ["conv1_pad", "conv1_conv", "pool1_pad", "pool1_pool"]
    assert names[-4:] == ["post_bn", "post_relu", "avg_pool", "predictions"]
    assert m.get_layer("conv1_conv").use_bias
    for b in ("conv2_block1", "conv3_block4"):
        for suffix in ("_preact_bn", "_preact_relu", "_1_conv", "_1_bn", "_1_relu", "_2_pad", "_2_conv", "_2_bn", "_2_relu",
                       "_3_conv", "_out"):
            assert b + suffix in names, b + suffix
        assert not m.get_layer(b + "_1_conv").use_bias and not m.get_layer(b + "_2_conv").use_bias
        assert m.get_layer(b + "_3_conv").use_bias
        assert m.get_layer(b + "_preact_bn").epsilon == 1.001e-5
    # the projection shortcut reads the pre-activation, only in the first block of a stack
    assert [n for n in names if n.endswith("_0_conv")] == [f"conv{s}_block1_0_conv" for s in (2, 3, 4, 5)]
    nodes = {l.name: ins for l, ins in m.iter_nodes()}
    assert nodes["conv2_block1_0_conv"] == ["conv2_block1_preact_relu"]
    # the strided last block of conv2..conv4: the stride is on _2_conv and the identity goes through MaxPooling2D(1, 2)
    pools = [l for l, _ in m.iter_nodes() if isinstance(l, K.MaxPooling2D) and l.name != "pool1_pool"]
    assert [(l.pool_size, l.strides) for l in pools] == [((1, 1), (2, 2))] * 3
    assert [nodes[l.name] for l in pools] == [["conv2_block2_out"], ["conv3_block3_out"], ["conv4_block5_out"]]
    assert m.get_layer("conv2_block3_2_conv").strides == (2, 2) and m.get_layer("conv5_block3_2_conv").strides == (1, 1)
    assert nodes["conv2_block3_out"] == [pools[0].name, "conv2_block3_3_conv"]


@pytest.mark.parametrize("name", list(V2))
def test_synthetic_probabilities_unsaturated(models, name):
    m = models[name]
    x = applications.synthetic_input(2, seed=0)
    p = torch_cpu.TorchCpuModel(m.to_json(), m.get_weights()).predict(x)
    assert np.allclose(p.sum(1), 1, atol=1e-4)
    assert p.max() <= 0.9, p.max(1)
    assert ((p > 1e-3).sum(1) >= 5).all(), (p > 1e-3).sum(1)
    # the residual stream stays O(1): the last Add and the pooled features
    feats = torch_cpu.TorchCpuModel(*_prefix(m, "avg_pool")).predict(x)
    assert 0.3 < np.sqrt((feats ** 2).mean()) < 10


def _prefix(m, last):
    part = dag_util.construct_model(m, m.input._keras_history[0].name, last, part_name="prefix")
    return part.to_json(), part.get_weights()


def test_existing_models_weights_unchanged(monkeypatch):
    """The V2 rule touches only convs that feed an Add directly: no V1 model or VGG16 has one, so their weights do not
    depend on it (ResNet50 seed 1 is also pinned bit for bit by tests/test_oracle_pin.py)."""
    for builder in (applications.ResNet50, applications.ResNet101, applications.ResNet152, applications.VGG16):
        want = builder().get_weights()
        monkeypatch.setattr(applications, "V2_BRANCH_GAIN", 123.0)
        got = builder().get_weights()
        monkeypatch.undo()
        assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want)), builder.__name__
    # ... while every V2 _3_conv kernel carries it, drawn from the same RNG stream
    m = applications.ResNet50V2()
    monkeypatch.setattr(applications, "V2_BRANCH_GAIN", 1.0)
    m1 = applications.ResNet50V2()
    k, k1 = m.get_layer("conv4_block2_3_conv").get_weights(), m1.get_layer("conv4_block2_3_conv").get_weights()
    assert np.allclose(k[0], k1[0] * 2.2, rtol=1e-6, atol=0) and not np.array_equal(k[0], k1[0])
    assert np.array_equal(k[1], k1[1])
    assert np.array_equal(m.get_layer("conv4_block2_2_conv").get_weights()[0], m1.get_layer("conv4_block2_2_conv").get_weights()[0])


@pytest.mark.parametrize("cuts", [["conv2_block3_out", "conv4_block1_out"],
                                  ["conv3_block1_preact_relu", "conv4_block6_out", "conv5_block1_preact_relu"]])
def test_partitions_compose_to_the_whole_model(models, cuts):
    m = models["ResNet50V2"]
    x = applications.synthetic_input(1, seed=4)
    names = [m.input._keras_history[0].name] + cuts + [m.output._keras_history[0].name]
    parts = [dag_util.construct_model(m, names[i], names[i + 1], part_name=f"p{i}") for i in range(len(names) - 1)]
    whole = keras_ref.predict(m.to_json(), m.get_weights(), x)
    piped = keras_ref.pipeline_predict([(p.to_json(), p.get_weights()) for p in parts], x)
    assert keras_ref.rel_err(piped, whole) <= 1e-6


def _bn(x, w, eps=1.001e-5):
    g, b, mean, var = (torch.from_numpy(a).double() for a in w)
    return F.batch_norm(x, mean, var, g, b, training=False, eps=eps)


def _conv(x, layer, stride=1):
    w = layer.get_weights()
    k = torch.from_numpy(w[0]).double().permute(3, 2, 0, 1)
    return F.conv2d(x, k, torch.from_numpy(w[1]).double() if len(w) > 1 else None, stride=stride)


@pytest.mark.parametrize("stride,conv_shortcut", [(1, True), (1, False), (2, False)])
def test_block2_restated_with_torch_functional(stride, conv_shortcut):
    """One pre-activation block, independently restated (fp64, NCHW), against the oracle's run of the same graph."""
    K.clear_session()
    inp = K.Input(shape=(14, 14, 256))
    out = applications._block2(inp, 64, stride=stride, conv_shortcut=conv_shortcut, name="b")
    m = K.Model(inp, out, name="block")
    applications.synthetic_weights(m, seed=7)
    x = applications.synthetic_input(2, (14, 14, 256), seed=8)
    L = m.get_layer
    t = torch.from_numpy(x).double().permute(0, 3, 1, 2)
    pre = F.relu(_bn(t, L("b_preact_bn").get_weights()))
    sc = _conv(pre, L("b_0_conv"), stride) if conv_shortcut else (F.max_pool2d(t, 1, stride) if stride > 1 else t)
    y = F.relu(_bn(_conv(pre, L("b_1_conv")), L("b_1_bn").get_weights()))
    y = F.relu(_bn(_conv(F.pad(y, (1, 1, 1, 1)), L("b_2_conv"), stride), L("b_2_bn").get_weights()))
    want = (sc + _conv(y, L("b_3_conv"))).permute(0, 2, 3, 1).numpy()
    got = keras_ref.predict(m.to_json(), m.get_weights(), x)
    assert got.shape == want.shape == (2, 14 // stride, 14 // stride, 256)
    assert keras_ref.rel_err(got, want) <= 1e-5
