"""Stand-ins for SAVi's belief-predictor networks (belief_predictor.py:65-80): torchvision's resnet18 with the 2-channel
stem, and a restatement of the SMT ``custom_resnet18`` written from its description (stem Conv2d(C, 16, 7, 1, 3) +
GroupNorm(16, 16) + ReLU, stages of two BasicBlocks at widths 16/32/64/128, stride 2 with a 1x1 conv + GroupNorm
downsample from stage 2, every norm GroupNorm(16, C), flatten, Linear(4608, n)), plus seeded randomisation of every
weight and norm so the norms are exercised."""
import torch
import torch.nn as nn


def tv_resnet18(n_out):
    import torchvision
    m = torchvision.models.resnet18(weights=None)
    m.conv1 = nn.Conv2d(2, 64, kernel_size=7, stride=2, padding=3, bias=False)
    m.fc = nn.Linear(512, n_out)
    return m.eval()


class Block(nn.Module):
    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, cout, 3, stride, 1, bias=False)
        self.bn1 = nn.GroupNorm(16, cout)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(cout, cout, 3, 1, 1, bias=False)
        self.bn2 = nn.GroupNorm(16, cout)
        self.downsample = None
        if stride != 1 or cin != cout:
            self.downsample = nn.Sequential(nn.Conv2d(cin, cout, 1, stride, bias=False), nn.GroupNorm(16, cout))

    def forward(self, x):
        y = self.relu(self.bn1(self.conv1(x)))
        y = self.bn2(self.conv2(y))
        return self.relu(y + (x if self.downsample is None else self.downsample(x)))


class SmtResNet(nn.Module):
    def __init__(self, in_channels, n_out=2, fc_in=4608):
        super().__init__()
        self.conv1 = nn.Conv2d(in_channels, 16, 7, 1, 3, bias=False)
        self.bn1 = nn.GroupNorm(16, 16)
        self.relu = nn.ReLU(inplace=True)
        cin = 16
        for s, cout in enumerate((16, 32, 64, 128)):
            stride = 1 if s == 0 else 2
            setattr(self, f"layer{s + 1}", nn.Sequential(Block(cin, cout, stride), Block(cout, cout, 1)))
            cin = cout
        self.fc = nn.Linear(fc_in, n_out)

    def forward(self, x):
        x = self.relu(self.bn1(self.conv1(x)))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(torch.flatten(x, 1))


def randomise(net, seed):
    """Seeded conv / fc weights at He scale, norm affine parameters around (1, 0), BatchNorm running statistics away
    from (0, 1)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, nn.Conv2d):
                fan_in = m.in_channels * m.kernel_size[0] * m.kernel_size[1]
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
            elif isinstance(m, nn.Linear):
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) / m.in_features ** 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g) * 0.1)
            elif isinstance(m, (nn.BatchNorm2d, nn.GroupNorm)):
                m.weight.copy_(1.0 + 0.3 * torch.randn(m.weight.shape, generator=g))
                m.bias.copy_(0.2 * torch.randn(m.bias.shape, generator=g))
                if isinstance(m, nn.BatchNorm2d):
                    m.running_mean.copy_(0.3 * torch.randn(m.running_mean.shape, generator=g))
                    m.running_var.copy_(0.5 + torch.rand(m.running_var.shape, generator=g))
    return net


def make_net(kind, seed=0):
    """'tv21' (label classifier), 'tv23' (offline location predictor), 'smt2' / 'smt23' (online location predictor
    without / with the category channels)."""
    net = tv_resnet18(int(kind[2:])) if kind.startswith("tv") else SmtResNet(int(kind[3:]))
    return randomise(net, seed).eval()


def smt_net(in_channels, hw, n_out=2, seed=0):
    """The SMT network for an ``hw = (H, W)`` observation: its fc takes the 128 H4 W4 features left after the three
    stride-2 stages."""
    h, w = hw
    for _ in range(3):
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return randomise(SmtResNet(in_channels, n_out, 128 * h * w), seed).eval()


def network_input(x, labels=None):
    """What the reference feeds the network: the permuted observation, with the category broadcast and concatenated
    (cnn_forward, belief_predictor.py:123-134)."""
    s = x.permute(0, 3, 1, 2)
    if labels is None:
        return s
    return torch.cat([s, labels.reshape(labels.shape + (1, 1)).expand(labels.shape + s.shape[-2:])], dim=1)
