"""MNIST MLP used by the cent / decent programs.

Reference: struct Model, /root/reference/dmnist/cent/cent.cpp:16-35 (duplicate in
dmnist/decent/decent.cpp:19-38): Linear(784,128) -> ReLU -> Linear(128,10) -> ReLU.
The ReLU on the logits is part of the model definition (SURVEY.md Q11) and is kept
by default; `relu_logits=False` gives the conventional head.
4 parameter tensors, 101 770 elements.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops.shadow import ShadowLinear


class MLP(nn.Module):
    def __init__(self, in_features: int = 784, hidden: int = 128, classes: int = 10,
                 relu_logits: bool = True):
        super().__init__()
        self.fc1 = ShadowLinear(in_features, hidden)
        self.fc2 = ShadowLinear(hidden, classes)
        self.relu_logits = relu_logits

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = x.reshape(x.shape[0], -1)
        if x.is_cuda and torch.is_autocast_enabled():
            # Linear(784,128)+bias+ReLU over the whole shard: wgmma kernel with fused epilogue
            from ..ops.linear_tc import linear_act
            w = self.fc1.w16 if self.fc1.w16 is not None else self.fc1.weight
            b = self.fc1.b16 if self.fc1.b16 is not None else self.fc1.bias
            x = linear_act(x, w, b, relu=True)
        else:
            x = F.relu(self.fc1(x))
        x = self.fc2(x)
        return F.relu(x) if self.relu_logits else x
