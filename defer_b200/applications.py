"""ResNet50 / ResNet152 / VGG16 builders with Keras layer names and Keras arithmetic.

The reference imports these from ``tensorflow.python.keras.applications``
(``test/test.py:3,14``, ``test/local_infer.py:3,8``).  Graphs follow
``keras_applications`` 1.0.8 (restated, not vendored - see SURVEY.md 8c):

* ``ResNet50``: old-style ``resnet50.py`` - stride on the first 1x1 conv and on the projection
  shortcut, conv biases, BN eps 1e-3, auto-named ``Add``/``Activation`` layers (tf.keras
  zero-based: ``add, add_1, ... add_15``), so the cut list of ``test/test.py:18`` applies verbatim.
* ``ResNet152``: ``resnet_common.py`` (``conv{s}_block{b}_{1,2,3}_conv``, ``_add``, ``_out``, eps 1.001e-5).
* ``ResNet50V2`` / ``ResNet101V2`` / ``ResNet152V2``: ``resnet_common.py``'s pre-activation blocks
  (``_preact_bn``, ``_preact_relu``, ``_0_conv`` in the first block of a stack, bias-free ``_1_conv`` / ``_2_conv``,
  the stride in the last block with an auto-named ``MaxPooling2D(1, strides=2)`` identity shortcut, ``_out`` Adds,
  ``post_bn``, ``post_relu``).
* ``VGG16``: ``block{i}_conv{j}`` (relu inside the conv), ``block{i}_pool``, ``flatten``, ``fc1``, ``fc2``,
  ``predictions``.

ImageNet weights are not available offline; ``weights='synthetic'`` draws seeded weights
(He-normal kernels, O(0.1) biases and BN shifts) that keep activations O(1) through the depth.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np

from . import keras_like as K
from .resize import INTERPOLATIONS, resize_image  # noqa: F401  (Keras load_img's resize, keep_aspect_ratio too, as Pillow)
from .jpeg import decode_jpeg  # noqa: F401  (Keras load_img's JPEG decode of baseline and progressive files, bit for bit as Pillow)
from .png import decode_png  # noqa: F401  (Keras load_img's PNG decode of non-interlaced files, bit for bit as Pillow)
from .image import decode_image  # noqa: F401  (either of the two, told by the file's first bytes as Pillow does)
from .keras_like import (Activation, Add, BatchNormalization, Conv2D, Dense, Flatten,
                         GlobalAveragePooling2D, Input, MaxPooling2D, Model, ZeroPadding2D)


# --------------------------------------------------------------------------- synthetic weights

#: ResNet V2 residual-branch gain: the conv that feeds an ``Add`` directly is scaled by this over sqrt(number of Adds).
#: Chosen on the CPU oracle at seed 1: top-1 probability 0.84 / 0.08 / 0.11 for 50V2 / 101V2 / 152V2, with 10+ classes
#: above 1e-3 and every ``_out`` sum of RMS 0.5-6; 2.5 already pushes 50V2 to 0.97.
V2_BRANCH_GAIN = 2.2


def synthetic_weights(model: Model, seed: int = 1, logit_std: float = 2.0) -> None:
    """Fill ``model`` with deterministic weights (see DESIGN.md "Synthetic data").

    conv / dense kernels: He-normal; biases N(0, 0.1); BN gamma U(0.8, 1.2), beta N(0, 0.1),
    mean N(0, 0.1), var U(0.8, 1.2).  The BN that feeds the main branch of a residual ``Add``
    gets gamma x 0.25 so the variance stays O(1) over 16-50 blocks; a conv that feeds an ``Add``
    directly (ResNet V2) gets its kernel x ``V2_BRANCH_GAIN / sqrt(#Adds)``; the last Dense is scaled
    so logits have std ~``logit_std`` (softmax not saturated).
    """
    rng = np.random.default_rng(seed)
    # BN layers directly feeding an Add together with a deeper path get damped
    damp = set()
    for layer, ins in model.iter_nodes():
        if isinstance(layer, Add) and ins:
            for n in ins:
                l = model.get_layer(n)
                if isinstance(l, BatchNormalization):
                    damp.add(l.name)
    # projection-shortcut BNs are not damped (they carry the identity signal)
    for layer, ins in model.iter_nodes():
        if isinstance(layer, BatchNormalization) and layer.name in damp and ins:
            src = model.get_layer(ins[0])
            if isinstance(src, Conv2D) and (layer.name.endswith("branch1") or layer.name.endswith("_0_bn")):
                damp.discard(layer.name)
    # ResNet V2: a residual branch ends in a conv feeding the Add directly (no BN to damp), and the pre-activation BN that
    # reads the sum does not normalise it, so the sum grows geometrically with depth (top-1 probability 1.0 unscaled).
    # No V1 model or VGG has such a conv, so their weights are unchanged.
    n_adds = sum(isinstance(l, Add) for l, _ in model.iter_nodes())
    res_convs = {n for l, ins in model.iter_nodes() if isinstance(l, Add) for n in ins
                 if isinstance(model.get_layer(n), Conv2D)}
    res_scale = np.float32(V2_BRANCH_GAIN / np.sqrt(max(n_adds, 1)))
    last_dense = None
    for layer, _ in model.iter_nodes():
        if isinstance(layer, Dense):
            last_dense = layer
    for layer in model.layers:
        if isinstance(layer, Conv2D):
            kh, kw = layer.kernel_size
            fan_in = kh * kw * layer.in_channels
            w = [rng.standard_normal((kh, kw, layer.in_channels, layer.filters), dtype=np.float32)
                 * np.float32(np.sqrt(2.0 / fan_in))]
            if layer.use_bias:
                w.append((rng.standard_normal(layer.filters, dtype=np.float32) * np.float32(0.1)))
            if layer.name in res_convs:
                w[0] = w[0] * res_scale     # after drawing: the RNG stream is the same with or without it
            layer.set_weights(w)
        elif isinstance(layer, Dense):
            fan_in = layer.in_features
            scale = np.sqrt(2.0 / fan_in)
            w = [rng.standard_normal((fan_in, layer.units), dtype=np.float32) * np.float32(scale)]
            if layer.use_bias:
                w.append(rng.standard_normal(layer.units, dtype=np.float32) * np.float32(0.1))
            layer.set_weights(w)
        elif isinstance(layer, BatchNormalization):
            c = layer.channels
            g = rng.uniform(0.8, 1.2, c).astype(np.float32)
            if layer.name in damp:
                g *= np.float32(0.25)
            layer.set_weights([g,
                               (rng.standard_normal(c) * 0.1).astype(np.float32),
                               (rng.standard_normal(c) * 0.1).astype(np.float32),
                               rng.uniform(0.8, 1.2, c).astype(np.float32)])
    if last_dense is not None and logit_std:
        # scale so that logits ~ N(0, logit_std^2) for O(1) inputs
        w = last_dense.get_weights()
        w[0] = w[0] * np.float32(logit_std / np.sqrt(2.0))
        last_dense.set_weights(w)


def synthetic_input(batch: int = 1, shape=(224, 224, 3), seed: int = 0) -> np.ndarray:
    """Seeded stand-in for the preprocessed image of ``test/test.py:19-23``."""
    rng = np.random.default_rng(seed)
    return rng.standard_normal((batch,) + tuple(shape), dtype=np.float32)


def synthetic_image(batch: int = 1, shape=(224, 224, 3), seed: int = 0) -> np.ndarray:
    """Seeded stand-in for ``img_to_array(load_img(...)).astype(np.uint8)``: uniform uint8 RGB, 0..255."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (batch,) + tuple(shape), dtype=np.uint8)


#: ImageNet channel means of Keras' caffe mode, in BGR order (keras_applications.imagenet_utils)
CAFFE_MEAN_BGR = (103.939, 116.779, 123.68)
#: the ``preprocess=`` modes of DEFER / StageRunner / plan_stage: Keras' ``preprocess_input`` of ResNet50 / 101 / 152 and
#: VGG16 ('caffe'), and of ResNet50V2 / 101V2 / 152V2 ('tf')
PREPROCESS_MODES = ("caffe", "tf")


def preprocess_input(x: np.ndarray, mode: str = "caffe") -> np.ndarray:
    """Keras ``preprocess_input`` of ResNet50 / ResNet101 / ResNet152 / VGG16 (caffe mode), channels-last, as the
    reference applies it before queueing an image (``test/test.py:23``).

    Restates ``keras_applications.imagenet_utils._preprocess_numpy_input``: non-float input becomes float32, the channel
    axis is reversed (RGB -> BGR) and the ImageNet mean is subtracted per channel in float32.  Returns a new float32
    array; ``x`` is not modified.  ``DEFER(..., preprocess="caffe")`` applies the same transform on the GPU.
    """
    if mode != "caffe":
        raise ValueError(f"preprocess_input(mode={mode!r}): this function applies 'caffe' mode only; "
                         "use resnet_v2_preprocess_input for 'tf' mode")
    x = np.asarray(x)
    if x.shape[-1] != 3:
        raise ValueError(f"preprocess_input: expected channels-last RGB (last axis 3), got shape {x.shape}")
    y = x[..., ::-1].astype(np.float32)          # astype copies: the caller's array is never touched
    y -= np.asarray(CAFFE_MEAN_BGR, np.float32)
    return y


def resnet_v2_preprocess_input(x: np.ndarray) -> np.ndarray:
    """Keras ``preprocess_input`` of ResNet50V2 / ResNet101V2 / ResNet152V2 (tf mode).

    Restates ``keras_applications.imagenet_utils._preprocess_numpy_input(x, mode='tf')``: non-float input becomes
    float32, then ``x /= 127.5; x -= 1.`` in float32 - no channel flip, no mean.  Returns a new float32 array; ``x`` is
    not modified.  ``DEFER(..., preprocess="tf")`` applies the same transform on the GPU, bit for bit.
    """
    y = np.asarray(x).astype(np.float32)        # astype copies: the caller's array is never touched
    y /= np.float32(127.5)
    y -= np.float32(1.0)
    return y


def caffe_shift() -> np.ndarray:
    """The per-channel shift the device applies after the channel flip: ``-float32(mean)``, BGR order."""
    return -np.asarray(CAFFE_MEAN_BGR, np.float32)


def check_preprocess(mode) -> None:
    if mode not in PREPROCESS_MODES:
        raise ValueError(f"preprocess={mode!r}: the supported modes are 'caffe' (Keras' preprocess_input of ResNet50/101/152 "
                         "and VGG16) and 'tf' (ResNet50V2/101V2/152V2)")


def check_model_preprocess(model, mode) -> None:
    """Refuse ``preprocess="tf"`` on a model whose Keras ``preprocess_input`` is caffe mode (``model.preprocess_mode``,
    recorded by the builders here).  A model without the record - a partition or one rebuilt from JSON - is not checked,
    and ``"caffe"`` stays accepted everywhere."""
    recorded = getattr(model, "preprocess_mode", None)
    if mode == "tf" and recorded == "caffe":
        raise ValueError(f"preprocess='tf': {model.name} is preprocessed in Keras' 'caffe' mode (RGB -> BGR, minus the "
                         "ImageNet mean); pass preprocess='caffe'")


def _finish(model: Model, weights: Optional[str], seed: int, preprocess_mode: str = "caffe") -> Model:
    model.preprocess_mode = preprocess_mode     # the mode of this model's Keras preprocess_input
    if weights in ("synthetic", "imagenet"):
        # 'imagenet' is accepted for script compatibility (test/test.py:14) but cannot be
        # downloaded offline: synthetic weights are used and flagged on the model.
        synthetic_weights(model, seed=seed)
        model.weights_source = "synthetic(seed=%d)" % seed
    elif weights is None:
        model.weights_source = "zeros"
    else:
        raise ValueError(f"weights={weights!r}: use 'synthetic' or None")
    return model


# --------------------------------------------------------------------------- ResNet50 (old-style)

def _identity_block(x, kernel_size, filters, stage, block):
    f1, f2, f3 = filters
    conv = f"res{stage}{block}_branch"
    bn = f"bn{stage}{block}_branch"
    y = Conv2D(f1, (1, 1), name=conv + "2a")(x)
    y = BatchNormalization(name=bn + "2a")(y)
    y = Activation("relu")(y)
    y = Conv2D(f2, kernel_size, padding="same", name=conv + "2b")(y)
    y = BatchNormalization(name=bn + "2b")(y)
    y = Activation("relu")(y)
    y = Conv2D(f3, (1, 1), name=conv + "2c")(y)
    y = BatchNormalization(name=bn + "2c")(y)
    y = Add()([y, x])
    return Activation("relu")(y)


def _conv_block(x, kernel_size, filters, stage, block, strides=(2, 2)):
    f1, f2, f3 = filters
    conv = f"res{stage}{block}_branch"
    bn = f"bn{stage}{block}_branch"
    y = Conv2D(f1, (1, 1), strides=strides, name=conv + "2a")(x)
    y = BatchNormalization(name=bn + "2a")(y)
    y = Activation("relu")(y)
    y = Conv2D(f2, kernel_size, padding="same", name=conv + "2b")(y)
    y = BatchNormalization(name=bn + "2b")(y)
    y = Activation("relu")(y)
    y = Conv2D(f3, (1, 1), name=conv + "2c")(y)
    y = BatchNormalization(name=bn + "2c")(y)
    sc = Conv2D(f3, (1, 1), strides=strides, name=conv + "1")(x)
    sc = BatchNormalization(name=bn + "1")(sc)
    y = Add()([y, sc])
    return Activation("relu")(y)


def ResNet50(weights: Optional[str] = "synthetic", include_top: bool = True, input_shape=(224, 224, 3),
             classes: int = 1000, seed: int = 1, fresh_names: bool = True) -> Model:
    if not include_top:
        raise ValueError("DEFER's scripts use include_top=True (test/test.py:14)")
    if fresh_names:
        K.clear_session()
    img = Input(shape=input_shape)
    x = ZeroPadding2D(padding=(3, 3), name="conv1_pad")(img)
    x = Conv2D(64, (7, 7), strides=(2, 2), padding="valid", name="conv1")(x)
    x = BatchNormalization(name="bn_conv1")(x)
    x = Activation("relu")(x)
    x = ZeroPadding2D(padding=(1, 1), name="pool1_pad")(x)
    x = MaxPooling2D((3, 3), strides=(2, 2))(x)
    x = _conv_block(x, 3, [64, 64, 256], 2, "a", strides=(1, 1))
    for b in "bc":
        x = _identity_block(x, 3, [64, 64, 256], 2, b)
    x = _conv_block(x, 3, [128, 128, 512], 3, "a")
    for b in "bcd":
        x = _identity_block(x, 3, [128, 128, 512], 3, b)
    x = _conv_block(x, 3, [256, 256, 1024], 4, "a")
    for b in "bcdef":
        x = _identity_block(x, 3, [256, 256, 1024], 4, b)
    x = _conv_block(x, 3, [512, 512, 2048], 5, "a")
    for b in "bc":
        x = _identity_block(x, 3, [512, 512, 2048], 5, b)
    x = GlobalAveragePooling2D(name="avg_pool")(x)
    x = Dense(classes, activation="softmax", name="fc1000")(x)
    return _finish(Model(img, x, name="resnet50"), weights, seed)


# --------------------------------------------------------------------------- ResNet152 (resnet_common)

def _block1(x, filters, kernel_size=3, stride=1, conv_shortcut=True, name=""):
    eps = 1.001e-5
    if conv_shortcut:
        sc = Conv2D(4 * filters, 1, strides=stride, name=name + "_0_conv")(x)
        sc = BatchNormalization(epsilon=eps, name=name + "_0_bn")(sc)
    else:
        sc = x
    y = Conv2D(filters, 1, strides=stride, name=name + "_1_conv")(x)
    y = BatchNormalization(epsilon=eps, name=name + "_1_bn")(y)
    y = Activation("relu", name=name + "_1_relu")(y)
    y = Conv2D(filters, kernel_size, padding="same", name=name + "_2_conv")(y)
    y = BatchNormalization(epsilon=eps, name=name + "_2_bn")(y)
    y = Activation("relu", name=name + "_2_relu")(y)
    y = Conv2D(4 * filters, 1, name=name + "_3_conv")(y)
    y = BatchNormalization(epsilon=eps, name=name + "_3_bn")(y)
    y = Add(name=name + "_add")([sc, y])
    return Activation("relu", name=name + "_out")(y)


def _stack1(x, filters, blocks, stride1=2, name=""):
    x = _block1(x, filters, stride=stride1, name=name + "_block1")
    for i in range(2, blocks + 1):
        x = _block1(x, filters, conv_shortcut=False, name=f"{name}_block{i}")
    return x


def _resnet_common(blocks, model_name, weights, input_shape, classes, seed, fresh_names):
    if fresh_names:
        K.clear_session()
    img = Input(shape=input_shape)
    x = ZeroPadding2D(padding=((3, 3), (3, 3)), name="conv1_pad")(img)
    x = Conv2D(64, 7, strides=2, name="conv1_conv")(x)
    x = BatchNormalization(epsilon=1.001e-5, name="conv1_bn")(x)
    x = Activation("relu", name="conv1_relu")(x)
    x = ZeroPadding2D(padding=((1, 1), (1, 1)), name="pool1_pad")(x)
    x = MaxPooling2D(3, strides=2, name="pool1_pool")(x)
    x = _stack1(x, 64, blocks[0], stride1=1, name="conv2")
    x = _stack1(x, 128, blocks[1], name="conv3")
    x = _stack1(x, 256, blocks[2], name="conv4")
    x = _stack1(x, 512, blocks[3], name="conv5")
    x = GlobalAveragePooling2D(name="avg_pool")(x)
    x = Dense(classes, activation="softmax", name="probs")(x)
    return _finish(Model(img, x, name=model_name), weights, seed)


def ResNet152(weights: Optional[str] = "synthetic", include_top: bool = True, input_shape=(224, 224, 3),
              classes: int = 1000, seed: int = 1, fresh_names: bool = True) -> Model:
    return _resnet_common([3, 8, 36, 3], "resnet152", weights, input_shape, classes, seed, fresh_names)


def ResNet101(weights: Optional[str] = "synthetic", include_top: bool = True, input_shape=(224, 224, 3),
              classes: int = 1000, seed: int = 1, fresh_names: bool = True) -> Model:
    return _resnet_common([3, 4, 23, 3], "resnet101", weights, input_shape, classes, seed, fresh_names)


# --------------------------------------------------------------------------- ResNet V2 (resnet_common, pre-activation)

def _block2(x, filters, kernel_size=3, stride=1, conv_shortcut=False, name=""):
    eps = 1.001e-5
    preact = BatchNormalization(epsilon=eps, name=name + "_preact_bn")(x)
    preact = Activation("relu", name=name + "_preact_relu")(preact)
    if conv_shortcut:
        sc = Conv2D(4 * filters, 1, strides=stride, name=name + "_0_conv")(preact)
    else:
        sc = MaxPooling2D(1, strides=stride)(x) if stride > 1 else x
    y = Conv2D(filters, 1, strides=1, use_bias=False, name=name + "_1_conv")(preact)
    y = BatchNormalization(epsilon=eps, name=name + "_1_bn")(y)
    y = Activation("relu", name=name + "_1_relu")(y)
    y = ZeroPadding2D(padding=((1, 1), (1, 1)), name=name + "_2_pad")(y)
    y = Conv2D(filters, kernel_size, strides=stride, use_bias=False, name=name + "_2_conv")(y)
    y = BatchNormalization(epsilon=eps, name=name + "_2_bn")(y)
    y = Activation("relu", name=name + "_2_relu")(y)
    y = Conv2D(4 * filters, 1, name=name + "_3_conv")(y)
    return Add(name=name + "_out")([sc, y])


def _stack2(x, filters, blocks, stride1=2, name=""):
    x = _block2(x, filters, conv_shortcut=True, name=name + "_block1")
    for i in range(2, blocks):
        x = _block2(x, filters, name=f"{name}_block{i}")
    return _block2(x, filters, stride=stride1, name=f"{name}_block{blocks}")


def _resnet_v2(blocks, model_name, weights, input_shape, classes, seed, fresh_names):
    if fresh_names:
        K.clear_session()
    img = Input(shape=input_shape)
    x = ZeroPadding2D(padding=((3, 3), (3, 3)), name="conv1_pad")(img)
    x = Conv2D(64, 7, strides=2, name="conv1_conv")(x)
    x = ZeroPadding2D(padding=((1, 1), (1, 1)), name="pool1_pad")(x)
    x = MaxPooling2D(3, strides=2, name="pool1_pool")(x)
    x = _stack2(x, 64, blocks[0], name="conv2")
    x = _stack2(x, 128, blocks[1], name="conv3")
    x = _stack2(x, 256, blocks[2], name="conv4")
    x = _stack2(x, 512, blocks[3], stride1=1, name="conv5")
    x = BatchNormalization(epsilon=1.001e-5, name="post_bn")(x)
    x = Activation("relu", name="post_relu")(x)
    x = GlobalAveragePooling2D(name="avg_pool")(x)
    x = Dense(classes, activation="softmax", name="predictions")(x)
    return _finish(Model(img, x, name=model_name), weights, seed, preprocess_mode="tf")


def ResNet50V2(weights: Optional[str] = "synthetic", include_top: bool = True, input_shape=(224, 224, 3),
               classes: int = 1000, seed: int = 1, fresh_names: bool = True) -> Model:
    return _resnet_v2([3, 4, 6, 3], "resnet50v2", weights, input_shape, classes, seed, fresh_names)


def ResNet101V2(weights: Optional[str] = "synthetic", include_top: bool = True, input_shape=(224, 224, 3),
                classes: int = 1000, seed: int = 1, fresh_names: bool = True) -> Model:
    return _resnet_v2([3, 4, 23, 3], "resnet101v2", weights, input_shape, classes, seed, fresh_names)


def ResNet152V2(weights: Optional[str] = "synthetic", include_top: bool = True, input_shape=(224, 224, 3),
                classes: int = 1000, seed: int = 1, fresh_names: bool = True) -> Model:
    return _resnet_v2([3, 8, 36, 3], "resnet152v2", weights, input_shape, classes, seed, fresh_names)


# --------------------------------------------------------------------------- VGG16

def VGG16(weights: Optional[str] = "synthetic", include_top: bool = True, input_shape=(224, 224, 3),
          classes: int = 1000, seed: int = 1, fresh_names: bool = True) -> Model:
    if fresh_names:
        K.clear_session()
    img = Input(shape=input_shape)
    x = img
    for bi, (n, f) in enumerate([(2, 64), (2, 128), (3, 256), (3, 512), (3, 512)], start=1):
        for ci in range(1, n + 1):
            x = Conv2D(f, (3, 3), activation="relu", padding="same", name=f"block{bi}_conv{ci}")(x)
        x = MaxPooling2D((2, 2), strides=(2, 2), name=f"block{bi}_pool")(x)
    x = Flatten(name="flatten")(x)
    x = Dense(4096, activation="relu", name="fc1")(x)
    x = Dense(4096, activation="relu", name="fc2")(x)
    x = Dense(classes, activation="softmax", name="predictions")(x)
    return _finish(Model(img, x, name="vgg16"), weights, seed)


# --------------------------------------------------------------------------- cut lists

def residual_add_names(model: Model) -> List[str]:
    """Names of the residual ``Add`` layers in execution order (legal cut points)."""
    return [l.name for l, _ in model.iter_nodes() if isinstance(l, Add)]


#: the cut list of reference ``test/test.py:18`` (tf.keras naming: Add layers add..add_15)
RESNET50_TEST_CUTS = ["add_2", "add_4", "add_6", "add_8", "add_10", "add_12", "add_14"]


def resolve_cut_names(model: Model, cuts: List[str], naming: str = "tf.keras") -> List[str]:
    """Map a user's cut list onto this model.  ``naming='keras'`` reads ``add_k`` one-based
    (standalone Keras auto-naming, ``add_1..add_16``) - see SURVEY.md 8a note."""
    if naming == "tf.keras":
        return list(cuts)
    if naming != "keras":
        raise ValueError(naming)
    adds = residual_add_names(model)
    out = []
    for c in cuts:
        if c.startswith("add_") and c[4:].isdigit():
            out.append(adds[int(c[4:]) - 1])
        else:
            out.append(c)
    return out


def default_cuts(model: Model, n_stages: int) -> List[str]:
    """Cut lists used by the BASELINE configs (SURVEY.md 8d) for 1/2/4/8 stages."""
    if n_stages <= 1:
        return []
    adds = residual_add_names(model)
    if model.name == "resnet50":
        table = {2: [6], 4: [2, 6, 12], 8: [2, 4, 6, 8, 10, 12, 14]}   # zero-based Add indices
        if n_stages in table:
            return [adds[i] for i in table[n_stages]]
    if model.name == "resnet152" and n_stages == 8:
        return [adds[i - 1] for i in (5, 11, 17, 23, 29, 35, 41)]
    if model.name == "vgg16" and n_stages == 4:
        return ["block1_pool", "block2_pool", "block3_pool"]
    if adds and n_stages - 1 <= len(adds):
        idx = np.linspace(0, len(adds), n_stages + 1)[1:-1]
        return [adds[int(round(i)) - 1] for i in idx]
    raise ValueError(f"no default cut list for {model.name} at {n_stages} stages")
