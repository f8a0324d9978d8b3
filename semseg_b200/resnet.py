"""Deep-stem dilated-ResNet backbone, drop-in for the reference's model/resnet.py.

Same public surface (`ResNet`, `Bottleneck`, `resnet50/101/152`, `pretrained=True` reading
`./initmodel/resnetNN_v2.pth` with strict=False — model/resnet.py:190-229) and the same child modules /
state_dict keys (real nn.Conv2d / nn.BatchNorm2d children, so nn.SyncBatchNorm.convert_sync_batchnorm and
DDP keep working, tool/train.py:141-157). Modules are constructed in the reference's order
(model/resnet.py:100-128), so a given torch.manual_seed yields bit-identical initial weights.

What differs is the execution: `forward_nhwc` runs on NHWC bf16 activations through the sm_90a kernels
(semseg_b200/functional.py); the nn.Conv2d / nn.BatchNorm2d children are parameter holders whose own
forward is never called. `BasicBlock` / resnet18/34 are unreachable from PSPNet/PSANet
(model/pspnet.py:32) and are not provided.
"""
import torch
import torch.nn as nn

from . import functional as SF

__all__ = ['ResNet', 'Bottleneck', 'resnet50', 'resnet101', 'resnet152']


def conv3x3(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


class NHWCSequential(nn.Sequential):
    """nn.Sequential whose children implement forward_nhwc (NHWC bf16 in/out)."""

    def forward_nhwc(self, x):
        for m in self:
            x = m.forward_nhwc(x)
        return x

    @SF.network_forward
    def forward(self, x):
        # standalone use with an fp32 NCHW tensor (the reference's calling convention)
        return SF.to_nchw_f32(self.forward_nhwc(SF.to_nhwc_bf16(x)))


class Bottleneck(nn.Module):
    """1x1 -> 3x3 (stride / dilation patched by the segmentation nets) -> 1x1, + residual (model/resnet.py:58-94)."""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super(Bottleneck, self).__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * self.expansion, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * self.expansion)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def forward_nhwc(self, x):
        return SF.bottleneck(x, self)

    @SF.network_forward
    def forward(self, x):
        return SF.to_nchw_f32(self.forward_nhwc(SF.to_nhwc_bf16(x)))


class Stem(NHWCSequential):
    """layer0 = conv1,bn1,relu,conv2,bn2,relu,conv3,bn3,relu,maxpool with the reference's child indices
    (model/pspnet.py:46) so state_dict keys are layer0.0.weight, layer0.1.weight, ..."""

    def forward_nhwc(self, x):
        return self._rest(SF.conv_bn_act(x, self[0], self[1], relu=True))

    def forward_nchw(self, x):
        """fp32 NCHW module input -> NHWC activation; when x needs a gradient it comes from the stem dgrad kernel."""
        return self._rest(SF.stem_conv_bn_act(x, self[0], self[1], relu=True))

    def _rest(self, x):
        x = SF.conv_bn_act(x, self[3], self[4], relu=True)
        x = SF.conv_bn_act(x, self[6], self[7], relu=True)
        return SF.maxpool_nhwc(x, self[9])

    @SF.network_forward
    def forward(self, x):
        return SF.to_nchw_f32(self.forward_nchw(x))


class ResNet(nn.Module):

    def __init__(self, block, layers, num_classes=1000, deep_base=True):
        super(ResNet, self).__init__()
        assert block is Bottleneck, "only the Bottleneck ResNets (50/101/152) are on the semseg hot path"
        assert deep_base, "PSPNet/PSANet use the deep-stem variant"
        self.deep_base = deep_base
        self.inplanes = 128
        self.conv1 = conv3x3(3, 64, stride=2)
        self.bn1 = nn.BatchNorm2d(64)
        self.conv2 = conv3x3(64, 64)
        self.bn2 = nn.BatchNorm2d(64)
        self.conv3 = conv3x3(64, 128)
        self.bn3 = nn.BatchNorm2d(128)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(block, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(block, 512, layers[3], stride=2)
        self.avgpool = nn.AvgPool2d(7, stride=1)
        self.fc = nn.Linear(512 * block.expansion, num_classes)

        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode='fan_out', nonlinearity='relu')
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * block.expansion, kernel_size=1, stride=stride, bias=False),
                nn.BatchNorm2d(planes * block.expansion),
            )
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes))
        return NHWCSequential(*layers)

    def stem(self):
        return Stem(self.conv1, self.bn1, self.relu, self.conv2, self.bn2, self.relu, self.conv3, self.bn3,
                    self.relu, self.maxpool)

    @SF.network_forward
    def forward(self, x):
        # ImageNet-classification forward of the reference (model/resnet.py:147-164); not on the segmentation path.
        y = self.stem().forward_nchw(x)
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            y = layer.forward_nhwc(y)
        y = SF.to_nchw_f32(y)
        y = self.avgpool(y)
        return self.fc(y.view(y.size(0), -1))


def _load_pretrained(model, path):
    model.load_state_dict(torch.load(path), strict=False)


def resnet50(pretrained=False, **kwargs):
    model = ResNet(Bottleneck, [3, 4, 6, 3], **kwargs)
    if pretrained:
        _load_pretrained(model, './initmodel/resnet50_v2.pth')
    return model


def resnet101(pretrained=False, **kwargs):
    model = ResNet(Bottleneck, [3, 4, 23, 3], **kwargs)
    if pretrained:
        _load_pretrained(model, './initmodel/resnet101_v2.pth')
    return model


def resnet152(pretrained=False, **kwargs):
    model = ResNet(Bottleneck, [3, 8, 36, 3], **kwargs)
    if pretrained:
        _load_pretrained(model, './initmodel/resnet152_v2.pth')
    return model
