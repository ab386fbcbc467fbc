"""2D backbone (ResNet trunk + 3 transposed-conv upsamplers + 1x1 head).

Host-side mirror of the reference backbone interface
(`/root/reference/mvn/models/pose_resnet.py:184-318` PoseResNet,
`:321-377` get_pose_net).  The module tree is laid out so that `state_dict()`
has exactly the reference key set (conv1, bn1, layer{1..4}.{i}.conv{1,2,3} /
bn{1,2,3} / downsample.{0,1}, deconv_layers.{0,1,3,4,6,7}, final_layer and the
optional {alg,vol}_confidences heads), so reference checkpoints load unchanged.

These modules only *hold parameters* and provide an autograd-capable torch
forward (backend="torch": training / CPU plumbing).  The product inference
path walks this tree once (see engine.py) and runs hand-written sm_90a
kernels instead.
"""
import torch
from torch import nn

BN_MOMENTUM = 0.1

# depth -> (block kind, blocks per stage); reference pose_resnet.py:177-181
RESNET_SPEC = {
    18: ("basic", (2, 2, 2, 2)),
    34: ("basic", (3, 4, 6, 3)),
    50: ("bottleneck", (3, 4, 6, 3)),
    101: ("bottleneck", (3, 4, 23, 3)),
    152: ("bottleneck", (3, 8, 36, 3)),
}


def _bn(c):
    return nn.BatchNorm2d(c, momentum=BN_MOMENTUM)


class ResidualUnit(nn.Module):
    """One residual unit of the trunk.

    kind="basic":       3x3(stride) - 3x3                    (expansion 1, ref :25-54)
    kind="bottleneck":  1x1 - 3x3(stride) - 1x1(x4)          (expansion 4, ref :57-95)
    kind="caffe":       1x1(stride) - 3x3 - 1x1(x4)          (expansion 4, ref :98-137)
    """

    def __init__(self, kind, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.kind = kind
        self.stride = stride
        if kind == "basic":
            self.expansion = 1
            self.conv1 = nn.Conv2d(inplanes, planes, 3, stride, 1, bias=False)
            self.bn1 = _bn(planes)
            self.conv2 = nn.Conv2d(planes, planes, 3, 1, 1, bias=False)
            self.bn2 = _bn(planes)
        else:
            self.expansion = 4
            s1, s2 = (stride, 1) if kind == "caffe" else (1, stride)
            self.conv1 = nn.Conv2d(inplanes, planes, 1, s1, 0, bias=False)
            self.bn1 = _bn(planes)
            self.conv2 = nn.Conv2d(planes, planes, 3, s2, 1, bias=False)
            self.bn2 = _bn(planes)
            self.conv3 = nn.Conv2d(planes, planes * 4, 1, bias=False)
            self.bn3 = _bn(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample

    def stages(self):
        """[(conv, bn)] in execution order -- consumed by the native planner."""
        out = [(self.conv1, self.bn1), (self.conv2, self.bn2)]
        if self.kind != "basic":
            out.append((self.conv3, self.bn3))
        return out

    def forward(self, x):
        shortcut = x if self.downsample is None else self.downsample(x)
        st = self.stages()
        y = x
        for i, (conv, bn) in enumerate(st):
            y = bn(conv(y))
            if i + 1 < len(st):
                y = self.relu(y)
        return self.relu(y + shortcut)


class ConfidenceHead(nn.Module):
    """Global-average-pool confidence head (reference :140-174)."""

    def __init__(self, in_channels, n_classes):
        super().__init__()
        self.features = nn.Sequential(
            nn.Conv2d(in_channels, 512, 3, 1, 1), _bn(512), nn.MaxPool2d(2), nn.ReLU(inplace=True),
            nn.Conv2d(512, 256, 3, 1, 1), _bn(256), nn.MaxPool2d(2), nn.ReLU(inplace=True),
        )
        self.head = nn.Sequential(
            nn.Linear(256, 512), nn.ReLU(inplace=True),
            nn.Linear(512, 256), nn.ReLU(inplace=True),
            nn.Linear(256, n_classes), nn.Sigmoid(),
        )

    def forward(self, x):
        x = self.features(x)
        return self.head(x.flatten(2).mean(dim=-1))


class PoseResNet(nn.Module):
    def __init__(self, kind, layers, num_joints, num_input_channels=3,
                 deconv_filters=(256, 256, 256), alg_confidences=False, vol_confidences=False):
        super().__init__()
        self.num_joints = num_joints
        self.kind = kind
        expansion = 1 if kind == "basic" else 4

        self.conv1 = nn.Conv2d(num_input_channels, 64, 7, 2, 3, bias=False)
        self.bn1 = _bn(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, 2, 1)

        inplanes = 64
        for i, (planes, n_blocks) in enumerate(zip((64, 128, 256, 512), layers)):
            stride = 1 if i == 0 else 2
            units = []
            for j in range(n_blocks):
                ds = None
                if j == 0 and (stride != 1 or inplanes != planes * expansion):
                    ds = nn.Sequential(nn.Conv2d(inplanes, planes * expansion, 1, stride, bias=False),
                                       _bn(planes * expansion))
                units.append(ResidualUnit(kind, inplanes, planes, stride if j == 0 else 1, ds))
                inplanes = planes * expansion
            setattr(self, "layer%d" % (i + 1), nn.Sequential(*units))

        if alg_confidences:
            self.alg_confidences = ConfidenceHead(512 * expansion, num_joints)
        if vol_confidences:
            self.vol_confidences = ConfidenceHead(512 * expansion, 32)

        up = []
        for planes in deconv_filters:  # k=4, s=2, p=1, no bias (reference :245-291)
            up += [nn.ConvTranspose2d(inplanes, planes, 4, 2, 1, 0, bias=False), _bn(planes), nn.ReLU(inplace=True)]
            inplanes = planes
        self.deconv_layers = nn.Sequential(*up)
        self.final_layer = nn.Conv2d(inplanes, num_joints, 1, 1, 0)

    def trunk(self, x):
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        return self.layer4(self.layer3(self.layer2(self.layer1(x))))

    def forward(self, x):
        """-> (heatmaps, features, alg_confidences, vol_confidences), reference :293-318."""
        x = self.trunk(x)
        alg = self.alg_confidences(x) if hasattr(self, "alg_confidences") else None
        vol = self.vol_confidences(x) if hasattr(self, "vol_confidences") else None
        features = self.deconv_layers(x)
        return self.final_layer(features), features, alg, vol


def get_pose_net(config, device="cuda:0"):
    """Same contract as reference pose_resnet.py:321-377 (config = config.model.backbone)."""
    kind, layers = RESNET_SPEC[config.num_layers]
    if config.style == "caffe":
        kind = "caffe"
    model = PoseResNet(kind, layers, config.num_joints,
                       alg_confidences=config.alg_confidences, vol_confidences=config.vol_confidences)

    if config.init_weights:
        print("Loading pretrained weights from: {}".format(config.checkpoint))
        own = model.state_dict()
        loaded = torch.load(config.checkpoint, map_location=device)
        loaded = loaded.get("state_dict", loaded)
        picked = {}
        for key, value in loaded.items():
            name = key.replace("module.", "")
            if name in own and value.shape == own[name].shape:
                picked[name] = value
            elif name in ("final_layer.weight", "final_layer.bias"):
                # joint count differs from the checkpoint: keep the overlapping filters (ref :352-368)
                print("Reiniting final layer:", key)
                fresh = torch.zeros_like(own[name])
                if fresh.dim() > 1:
                    nn.init.xavier_uniform_(fresh)
                n = min(fresh.shape[0], value.shape[0])
                fresh[:n] = value[:n]
                picked[name] = fresh
        missing = {k.replace("module.", "") for k in loaded} - set(picked)
        if missing:
            print("Parameters [{}] were not inited".format(missing))
        model.load_state_dict(picked, strict=False)
        print("Successfully loaded pretrained weights for backbone")
    return model
