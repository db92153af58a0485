from .resnet import ResNet, BasicBlock, Bottleneck, resnet18, resnet34, resnet50, resnet101, resnet152
from .xception import Xception, xception39
