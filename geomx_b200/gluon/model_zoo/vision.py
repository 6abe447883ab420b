"""Vision models (parity: ``python/mxnet/gluon/model_zoo/vision/{alexnet,vgg,resnet,densenet,squeezenet,inception,mobilenet}.py`` — every name
of the reference's ``get_model`` table: resnet{18,34,50,101,152}_v{1,2}, vgg{11,13,16,19}[_bn], alexnet, densenet{121,161,169,201},
squeezenet1.{0,1}, inceptionv3, mobilenet{1.0,0.75,0.5,0.25}, mobilenetv2_*; same layer recipes, built from
``gluon.nn`` so that Conv/Dense/Pool/BatchNorm run through the native kernels on CUDA)."""
from __future__ import annotations

from ...base import MXNetError
from .. import nn
from ..block import HybridBlock

__all__ = ["get_model", "get_vgg", "get_resnet", "get_densenet", "get_mobilenet", "get_mobilenet_v2", "AlexNet", "alexnet", "VGG", "ResNetV1",
           "ResNetV2", "BasicBlockV1", "BasicBlockV2", "BottleneckV1", "BottleneckV2", "DenseNet", "SqueezeNet", "squeezenet1_0", "squeezenet1_1",
           "Inception3", "inception_v3", "MobileNet", "MobileNetV2", "LeNet", "lenet", "MLP", "mlp"]


class LeNet(HybridBlock):
    """The GeoMX demo CNN family (examples/cnn.py: Conv-Pool-Conv-Pool-Dense-Dense-Dense)."""

    def __init__(self, classes=10, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            self.features = nn.HybridSequential(prefix="")
            self.features.add(nn.Conv2D(16, 5, activation="relu"), nn.MaxPool2D(2, 2), nn.Conv2D(32, 5, activation="relu"), nn.MaxPool2D(2, 2), nn.Flatten(),
                              nn.Dense(256, activation="relu"), nn.Dense(128, activation="relu"))
            self.output = nn.Dense(classes)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class MLP(HybridBlock):
    def __init__(self, hidden=(512, 256), classes=10, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            self.features = nn.HybridSequential(prefix="")
            self.features.add(nn.Flatten())
            for h in hidden:
                self.features.add(nn.Dense(h, activation="relu"))
            self.output = nn.Dense(classes)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class AlexNet(HybridBlock):
    def __init__(self, classes=1000, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="")
            f.add(nn.Conv2D(64, 11, 4, 2, activation="relu"), nn.MaxPool2D(3, 2), nn.Conv2D(192, 5, padding=2, activation="relu"), nn.MaxPool2D(3, 2),
                  nn.Conv2D(384, 3, padding=1, activation="relu"), nn.Conv2D(256, 3, padding=1, activation="relu"),
                  nn.Conv2D(256, 3, padding=1, activation="relu"), nn.MaxPool2D(3, 2), nn.Flatten(), nn.Dense(4096, activation="relu"), nn.Dropout(0.5),
                  nn.Dense(4096, activation="relu"), nn.Dropout(0.5))
            self.output = nn.Dense(classes)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class VGG(HybridBlock):
    def __init__(self, layers, filters, classes=1000, batch_norm=False, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="")
            for n, c in zip(layers, filters):
                for _ in range(n):
                    f.add(nn.Conv2D(c, 3, padding=1))
                    if batch_norm:
                        f.add(nn.BatchNorm())
                    f.add(nn.Activation("relu"))
                f.add(nn.MaxPool2D(2, 2))
            f.add(nn.Flatten(), nn.Dense(4096, activation="relu"), nn.Dropout(0.5), nn.Dense(4096, activation="relu"), nn.Dropout(0.5))
            self.output = nn.Dense(classes)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class BasicBlockV1(HybridBlock):
    def __init__(self, channels, stride, downsample=False, in_channels=0, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            self.body = nn.HybridSequential(prefix="")
            self.body.add(nn.Conv2D(channels, 3, stride, 1, use_bias=False, in_channels=in_channels), nn.BatchNorm(), nn.Activation("relu"),
                          nn.Conv2D(channels, 3, 1, 1, use_bias=False, in_channels=channels), nn.BatchNorm())
            self.downsample = None
            if downsample:
                self.downsample = nn.HybridSequential(prefix="")
                self.downsample.add(nn.Conv2D(channels, 1, stride, use_bias=False, in_channels=in_channels), nn.BatchNorm())

    def hybrid_forward(self, F, x):
        res = x if self.downsample is None else self.downsample(x)
        return (self.body(x) + res).relu()


class BottleneckV1(HybridBlock):
    """1x1 → 3x3 → 1x1 residual unit of ResNet-50/101/152 (resnet.py BottleneckV1; the stride sits on the first 1x1 like the reference)."""

    def __init__(self, channels, stride, downsample=False, in_channels=0, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            self.body = nn.HybridSequential(prefix="")
            self.body.add(nn.Conv2D(channels // 4, 1, stride, use_bias=False), nn.BatchNorm(), nn.Activation("relu"),
                          nn.Conv2D(channels // 4, 3, 1, 1, use_bias=False), nn.BatchNorm(), nn.Activation("relu"),
                          nn.Conv2D(channels, 1, 1, use_bias=False), nn.BatchNorm())
            self.downsample = None
            if downsample:
                self.downsample = nn.HybridSequential(prefix="")
                self.downsample.add(nn.Conv2D(channels, 1, stride, use_bias=False, in_channels=in_channels), nn.BatchNorm())

    def hybrid_forward(self, F, x):
        res = x if self.downsample is None else self.downsample(x)
        return (self.body(x) + res).relu()


class BasicBlockV2(HybridBlock):
    """Pre-activation basic unit (He et al. 2016, resnet.py BasicBlockV2)."""

    def __init__(self, channels, stride, downsample=False, in_channels=0, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            self.bn1 = nn.BatchNorm(); self.conv1 = nn.Conv2D(channels, 3, stride, 1, use_bias=False, in_channels=in_channels)
            self.bn2 = nn.BatchNorm(); self.conv2 = nn.Conv2D(channels, 3, 1, 1, use_bias=False, in_channels=channels)
            self.downsample = nn.Conv2D(channels, 1, stride, use_bias=False, in_channels=in_channels) if downsample else None

    def hybrid_forward(self, F, x):
        residual = x
        x = self.bn1(x).relu()
        if self.downsample is not None:
            residual = self.downsample(x)
        x = self.conv1(x)
        x = self.conv2(self.bn2(x).relu())
        return x + residual


class BottleneckV2(HybridBlock):
    def __init__(self, channels, stride, downsample=False, in_channels=0, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            self.bn1 = nn.BatchNorm(); self.conv1 = nn.Conv2D(channels // 4, 1, 1, use_bias=False)
            self.bn2 = nn.BatchNorm(); self.conv2 = nn.Conv2D(channels // 4, 3, stride, 1, use_bias=False)
            self.bn3 = nn.BatchNorm(); self.conv3 = nn.Conv2D(channels, 1, 1, use_bias=False)
            self.downsample = nn.Conv2D(channels, 1, stride, use_bias=False, in_channels=in_channels) if downsample else None

    def hybrid_forward(self, F, x):
        residual = x
        x = self.bn1(x).relu()
        if self.downsample is not None:
            residual = self.downsample(x)
        x = self.conv1(x)
        x = self.conv2(self.bn2(x).relu())
        x = self.conv3(self.bn3(x).relu())
        return x + residual


class ResNetV2(HybridBlock):
    def __init__(self, block, layers, channels, classes=1000, thumbnail=False, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="")
            f.add(nn.BatchNorm(scale=False, center=False))
            if thumbnail:
                f.add(nn.Conv2D(channels[0], 3, 1, 1, use_bias=False))
            else:
                f.add(nn.Conv2D(channels[0], 7, 2, 3, use_bias=False), nn.BatchNorm(), nn.Activation("relu"), nn.MaxPool2D(3, 2, 1))
            cin = channels[0]
            for i, n in enumerate(layers):
                stride = 1 if i == 0 else 2
                f.add(block(channels[i + 1], stride, channels[i + 1] != cin, in_channels=cin))
                cin = channels[i + 1]
                for _ in range(n - 1):
                    f.add(block(channels[i + 1], 1, False, in_channels=cin))
            f.add(nn.BatchNorm(), nn.Activation("relu"), nn.GlobalAvgPool2D(), nn.Flatten())
            self.output = nn.Dense(classes, in_units=cin)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class ResNetV1(HybridBlock):
    def __init__(self, layers, channels, classes=1000, thumbnail=False, block=None, **kwargs):
        super().__init__(**kwargs)
        BasicBlockV1_ = block or BasicBlockV1
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="")
            if thumbnail:
                f.add(nn.Conv2D(channels[0], 3, 1, 1, use_bias=False))
            else:
                f.add(nn.Conv2D(channels[0], 7, 2, 3, use_bias=False), nn.BatchNorm(), nn.Activation("relu"), nn.MaxPool2D(3, 2, 1))
            for i, n in enumerate(layers):
                stride = 1 if i == 0 else 2
                f.add(BasicBlockV1_(channels[i + 1], stride, channels[i + 1] != channels[i] or stride != 1, in_channels=channels[i]))
                for _ in range(n - 1):
                    f.add(BasicBlockV1_(channels[i + 1], 1, False, in_channels=channels[i + 1]))
            f.add(nn.GlobalAvgPool2D(), nn.Flatten())
            self.output = nn.Dense(classes)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class _Fire(HybridBlock):
    def __init__(self, squeeze, e1, e3, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            self.squeeze = nn.Conv2D(squeeze, 1, activation="relu")
            self.e1 = nn.Conv2D(e1, 1, activation="relu")
            self.e3 = nn.Conv2D(e3, 3, padding=1, activation="relu")

    def hybrid_forward(self, F, x):
        s = self.squeeze(x)
        return F.concat(self.e1(s), self.e3(s), dim=1)


class SqueezeNet(HybridBlock):
    def __init__(self, version="1.1", classes=1000, **kwargs):
        super().__init__(**kwargs)
        assert version in ("1.0", "1.1"), "Unsupported SqueezeNet version %s: 1.0 or 1.1 expected" % version
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="")
            if version == "1.0":
                f.add(nn.Conv2D(96, 7, 2, activation="relu"), nn.MaxPool2D(3, 2, ceil_mode=True), _Fire(16, 64, 64), _Fire(16, 64, 64), _Fire(32, 128, 128),
                      nn.MaxPool2D(3, 2, ceil_mode=True), _Fire(32, 128, 128), _Fire(48, 192, 192), _Fire(48, 192, 192), _Fire(64, 256, 256),
                      nn.MaxPool2D(3, 2, ceil_mode=True), _Fire(64, 256, 256), nn.Dropout(0.5))
            else:
                f.add(nn.Conv2D(64, 3, 2, activation="relu"), nn.MaxPool2D(3, 2, ceil_mode=True), _Fire(16, 64, 64), _Fire(16, 64, 64),
                      nn.MaxPool2D(3, 2, ceil_mode=True), _Fire(32, 128, 128), _Fire(32, 128, 128), nn.MaxPool2D(3, 2, ceil_mode=True),
                      _Fire(48, 192, 192), _Fire(48, 192, 192), _Fire(64, 256, 256), _Fire(64, 256, 256), nn.Dropout(0.5))
            self.output = nn.HybridSequential(prefix="")
            self.output.add(nn.Conv2D(classes, 1, activation="relu"), nn.GlobalAvgPool2D(), nn.Flatten())

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class MobileNet(HybridBlock):
    def __init__(self, multiplier=1.0, classes=1000, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="")

            def conv(c, k=1, s=1, p=0, g=1, cin=0):
                f.add(nn.Conv2D(c, k, s, p, groups=g, use_bias=False, in_channels=cin), nn.BatchNorm(), nn.Activation("relu"))
            c0 = int(32 * multiplier)
            conv(c0, 3, 2, 1, cin=0)
            dw = [int(x * multiplier) for x in [32, 64] + [128] * 2 + [256] * 2 + [512] * 6 + [1024]]
            pw = [int(x * multiplier) for x in [64] + [128] * 2 + [256] * 2 + [512] * 6 + [1024] * 2]
            strides = [1, 2] * 3 + [1] * 5 + [2, 1]
            for d, c, s in zip(dw, pw, strides):
                conv(d, 3, s, 1, g=d, cin=d)
                conv(c, cin=d)
            f.add(nn.GlobalAvgPool2D(), nn.Flatten())
            self.output = nn.Dense(classes)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class _DenseLayer(HybridBlock):
    def __init__(self, growth_rate, bn_size, dropout, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            b = self.body = nn.HybridSequential(prefix="")
            b.add(nn.BatchNorm(), nn.Activation("relu"), nn.Conv2D(bn_size * growth_rate, 1, use_bias=False), nn.BatchNorm(), nn.Activation("relu"),
                  nn.Conv2D(growth_rate, 3, padding=1, use_bias=False))
            if dropout:
                b.add(nn.Dropout(dropout))

    def hybrid_forward(self, F, x):
        return F.concat(x, self.body(x), dim=1)


class DenseNet(HybridBlock):
    """Densely connected network (densenet.py): dense blocks of BN-ReLU-1x1-BN-ReLU-3x3 layers whose outputs are concatenated, transition
    layers (1x1 conv + 2x2 average pool) halve the channels in between."""

    def __init__(self, num_init_features, growth_rate, block_config, bn_size=4, dropout=0, classes=1000, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="")
            f.add(nn.Conv2D(num_init_features, 7, 2, 3, use_bias=False), nn.BatchNorm(), nn.Activation("relu"), nn.MaxPool2D(3, 2, 1))
            nf = num_init_features
            for i, n in enumerate(block_config):
                for _ in range(n):
                    f.add(_DenseLayer(growth_rate, bn_size, dropout))
                nf += n * growth_rate
                if i != len(block_config) - 1:
                    nf //= 2
                    f.add(nn.BatchNorm(), nn.Activation("relu"), nn.Conv2D(nf, 1, use_bias=False), nn.AvgPool2D(2, 2))
            f.add(nn.BatchNorm(), nn.Activation("relu"), nn.GlobalAvgPool2D(), nn.Flatten())
            self.output = nn.Dense(classes)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


def _conv_bn(channels, kernel, stride=1, pad=0):
    blk = nn.HybridSequential(prefix="")
    blk.add(nn.Conv2D(channels, kernel, stride, pad, use_bias=False), nn.BatchNorm(epsilon=0.001), nn.Activation("relu"))
    return blk


class _Branches(HybridBlock):
    """Parallel branches concatenated along the channel axis (the ``HybridConcurrent`` of inception.py)."""

    def __init__(self, branches, **kwargs):
        super().__init__(**kwargs)
        self._n = len(branches)
        for i, b in enumerate(branches):
            setattr(self, "b%d" % i, b)

    def hybrid_forward(self, F, x):
        return F.concat(*[getattr(self, "b%d" % i)(x) for i in range(self._n)], dim=1)


def _seq(*blocks):
    s = nn.HybridSequential(prefix="")
    s.add(*blocks)
    return s


def _inc_a(pool_features):
    return _Branches([_conv_bn(64, 1), _seq(_conv_bn(48, 1), _conv_bn(64, 5, 1, 2)), _seq(_conv_bn(64, 1), _conv_bn(96, 3, 1, 1), _conv_bn(96, 3, 1, 1)),
                      _seq(nn.AvgPool2D(3, 1, 1), _conv_bn(pool_features, 1))])


def _inc_b():
    return _Branches([_conv_bn(384, 3, 2), _seq(_conv_bn(64, 1), _conv_bn(96, 3, 1, 1), _conv_bn(96, 3, 2)), nn.MaxPool2D(3, 2)])


def _inc_c(c7):
    return _Branches([_conv_bn(192, 1), _seq(_conv_bn(c7, 1), _conv_bn(c7, (1, 7), 1, (0, 3)), _conv_bn(192, (7, 1), 1, (3, 0))),
                      _seq(_conv_bn(c7, 1), _conv_bn(c7, (7, 1), 1, (3, 0)), _conv_bn(c7, (1, 7), 1, (0, 3)), _conv_bn(c7, (7, 1), 1, (3, 0)),
                           _conv_bn(192, (1, 7), 1, (0, 3))),
                      _seq(nn.AvgPool2D(3, 1, 1), _conv_bn(192, 1))])


def _inc_d():
    return _Branches([_seq(_conv_bn(192, 1), _conv_bn(320, 3, 2)),
                      _seq(_conv_bn(192, 1), _conv_bn(192, (1, 7), 1, (0, 3)), _conv_bn(192, (7, 1), 1, (3, 0)), _conv_bn(192, 3, 2)), nn.MaxPool2D(3, 2)])


def _inc_e():
    return _Branches([_conv_bn(320, 1),
                      _seq(_conv_bn(384, 1), _Branches([_conv_bn(384, (1, 3), 1, (0, 1)), _conv_bn(384, (3, 1), 1, (1, 0))])),
                      _seq(_conv_bn(448, 1), _conv_bn(384, 3, 1, 1), _Branches([_conv_bn(384, (1, 3), 1, (0, 1)), _conv_bn(384, (3, 1), 1, (1, 0))])),
                      _seq(nn.AvgPool2D(3, 1, 1), _conv_bn(192, 1))])


class Inception3(HybridBlock):
    """Inception v3 (inception.py): 299x299 input, factorised 7x7 / 3x3 convolutions."""

    def __init__(self, classes=1000, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="")
            f.add(_conv_bn(32, 3, 2), _conv_bn(32, 3), _conv_bn(64, 3, 1, 1), nn.MaxPool2D(3, 2), _conv_bn(80, 1), _conv_bn(192, 3), nn.MaxPool2D(3, 2),
                  _inc_a(32), _inc_a(64), _inc_a(64), _inc_b(), _inc_c(128), _inc_c(160), _inc_c(160), _inc_c(192), _inc_d(), _inc_e(), _inc_e(),
                  nn.GlobalAvgPool2D(), nn.Dropout(0.5), nn.Flatten())
            self.output = nn.Dense(classes)

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


class _LinearBottleneck(HybridBlock):
    """MobileNetV2 inverted residual: 1x1 expand (ReLU6) → 3x3 depthwise (ReLU6) → 1x1 linear projection, identity shortcut when the shape
    is unchanged."""

    def __init__(self, in_channels, channels, t, stride, **kwargs):
        super().__init__(**kwargs)
        self.use_shortcut = stride == 1 and in_channels == channels
        with self.name_scope():
            o = self.out = nn.HybridSequential(prefix="")
            o.add(nn.Conv2D(in_channels * t, 1, use_bias=False), nn.BatchNorm(), nn.HybridLambda(lambda F, x: x.clip(0, 6)),
                  nn.Conv2D(in_channels * t, 3, stride, 1, groups=in_channels * t, use_bias=False), nn.BatchNorm(), nn.HybridLambda(lambda F, x: x.clip(0, 6)),
                  nn.Conv2D(channels, 1, use_bias=False), nn.BatchNorm())

    def hybrid_forward(self, F, x):
        out = self.out(x)
        return out + x if self.use_shortcut else out


class MobileNetV2(HybridBlock):
    def __init__(self, multiplier=1.0, classes=1000, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            f = self.features = nn.HybridSequential(prefix="features_")
            c0 = int(32 * multiplier)
            f.add(nn.Conv2D(c0, 3, 2, 1, use_bias=False), nn.BatchNorm(), nn.HybridLambda(lambda F, x: x.clip(0, 6)))
            in_group = [int(x * multiplier) for x in [32] + [16] + [24] * 2 + [32] * 3 + [64] * 4 + [96] * 3 + [160] * 3]
            out_group = [int(x * multiplier) for x in [16] + [24] * 2 + [32] * 3 + [64] * 4 + [96] * 3 + [160] * 3 + [320]]
            ts = [1] + [6] * 16
            strides = [1, 2] * 2 + [1, 1, 2] + [1] * 6 + [2] + [1] * 3
            for cin, c, t, s_ in zip(in_group, out_group, ts, strides):
                f.add(_LinearBottleneck(cin, c, t, s_))
            last = int(1280 * multiplier) if multiplier > 1.0 else 1280
            f.add(nn.Conv2D(last, 1, use_bias=False), nn.BatchNorm(), nn.HybridLambda(lambda F, x: x.clip(0, 6)), nn.GlobalAvgPool2D())
            self.output = nn.HybridSequential(prefix="output_")
            self.output.add(nn.Conv2D(classes, 1, use_bias=False), nn.Flatten())

    def hybrid_forward(self, F, x):
        return self.output(self.features(x))


_VGG = {11: [1, 1, 2, 2, 2], 13: [2, 2, 2, 2, 2], 16: [2, 2, 3, 3, 3], 19: [2, 2, 4, 4, 4]}
_RES = {18: ("basic", [2, 2, 2, 2], [64, 64, 128, 256, 512]), 34: ("basic", [3, 4, 6, 3], [64, 64, 128, 256, 512]),
        50: ("bottle", [3, 4, 6, 3], [64, 256, 512, 1024, 2048]), 101: ("bottle", [3, 4, 23, 3], [64, 256, 512, 1024, 2048]),
        152: ("bottle", [3, 8, 36, 3], [64, 256, 512, 1024, 2048])}
_DENSE = {121: (64, 32, [6, 12, 24, 16]), 161: (96, 48, [6, 12, 36, 24]), 169: (64, 32, [6, 12, 32, 32]), 201: (64, 32, [6, 12, 48, 32])}


def get_vgg(num_layers, batch_norm=False, **kw): return VGG(_VGG[num_layers], [64, 128, 256, 512, 512], batch_norm=batch_norm, **kw)


def get_resnet(version, num_layers, **kw):
    kind, layers, channels = _RES[num_layers]
    if version == 1:
        return ResNetV1(layers, channels, block=BasicBlockV1 if kind == "basic" else BottleneckV1, **kw)
    assert version == 2, "Invalid resnet version: %s. Options are 1 and 2." % version
    return ResNetV2(BasicBlockV2 if kind == "basic" else BottleneckV2, layers, channels, **kw)


def get_densenet(num_layers, **kw):
    init, growth, cfg = _DENSE[num_layers]
    return DenseNet(init, growth, cfg, **kw)


def get_mobilenet(multiplier, **kw): return MobileNet(multiplier, **kw)
def get_mobilenet_v2(multiplier, **kw): return MobileNetV2(multiplier, **kw)


def lenet(**kw): return LeNet(**kw)
def mlp(**kw): return MLP(**kw)
def alexnet(**kw): return AlexNet(**kw)
def squeezenet1_0(**kw): return SqueezeNet("1.0", **kw)
def squeezenet1_1(**kw): return SqueezeNet("1.1", **kw)
def inception_v3(**kw): return Inception3(**kw)


_models = {"lenet": lenet, "mlp": mlp, "alexnet": alexnet, "squeezenet1.0": squeezenet1_0, "squeezenet1.1": squeezenet1_1, "inceptionv3": inception_v3}


def _register_families():
    g = globals()
    for n in _VGG:
        for bn in (False, True):
            name = "vgg%d%s" % (n, "_bn" if bn else "")
            g[name] = (lambda n=n, bn=bn: lambda **kw: get_vgg(n, bn, **kw))(); _models[name] = g[name]
    for v in (1, 2):
        for n in _RES:
            name = "resnet%d_v%d" % (n, v)
            g[name] = (lambda v=v, n=n: lambda **kw: get_resnet(v, n, **kw))(); _models[name] = g[name]
    for n in _DENSE:
        name = "densenet%d" % n
        g[name] = (lambda n=n: lambda **kw: get_densenet(n, **kw))(); _models[name] = g[name]
    for m in (1.0, 0.75, 0.5, 0.25):
        tag = ("%g" % m) if m != 1.0 else "1.0"
        g["mobilenet" + tag.replace(".", "_")] = (lambda m=m: lambda **kw: get_mobilenet(m, **kw))(); _models["mobilenet" + tag] = g["mobilenet" + tag.replace(".", "_")]
        g["mobilenet_v2_" + tag.replace(".", "_")] = (lambda m=m: lambda **kw: get_mobilenet_v2(m, **kw))(); _models["mobilenetv2_" + tag] = g["mobilenet_v2_" + tag.replace(".", "_")]


_register_families()


def get_model(name, pretrained=False, **kwargs):
    if pretrained:
        # no download: the file must already be in the model store (model_store.get_model_file explains where it looked)
        from .model_store import get_model_file
        path = get_model_file(name, root=kwargs.pop("root", None))
        net = get_model(name, pretrained=False, **{k: v for k, v in kwargs.items() if k != "ctx"})
        net.load_parameters(path, ctx=kwargs.get("ctx"))
        return net
    name = name.lower()
    if name not in _models:
        raise MXNetError("Model %s is not supported. Available: %s" % (name, ", ".join(sorted(_models))))
    return _models[name](**kwargs)
