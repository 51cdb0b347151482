"""Seeded synthetic bilevel problems of the five shapes named in BASELINE.json / SURVEY.md §8(d).

Every factory builds its tensors on the CPU generator (``torch.manual_seed``) and then moves them to
the requested device, so the CPU oracle and the CUDA engine see bit-identical inputs.  The loss
structures restate the reference examples (cited per factory); models use default module init.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Callable, Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from .shim import ShimConfig, ShimProblem


@dataclass
class Workload:
    name: str
    lower: ShimProblem
    upper: ShimProblem
    vector: Tuple[torch.Tensor, ...]  # direction v, one tensor per lower parameter
    describe: dict


# ------------------------------------------------------------------------------------------------
# modules
# ------------------------------------------------------------------------------------------------
class LogisticWeights(nn.Module):
    """20-vector of logistic-regression weights (reference ``test/test_regression.py:13-22``)."""

    def __init__(self, dim=20):
        super().__init__()
        self.w = nn.Parameter(torch.zeros(dim))

    def forward(self, inputs):
        return inputs @ self.w, self.w


class DecayCoefficients(nn.Module):
    """Per-weight decay coefficients, the upper variable (reference ``test/test_regression.py:24-31``)."""

    def __init__(self, dim=20):
        super().__init__()
        self.w = nn.Parameter(torch.ones(dim))

    def forward(self):
        return self.w


class LeNet5(nn.Module):
    """Canonical LeNet-5 on 3x32x32 (SURVEY §0 item 2: stands in for the example's ResNet32)."""

    def __init__(self, num_classes=10):
        super().__init__()
        self.features = nn.Sequential(
            nn.Conv2d(3, 6, 5), nn.ReLU(), nn.MaxPool2d(2),
            nn.Conv2d(6, 16, 5), nn.ReLU(), nn.MaxPool2d(2),
        )
        self.classifier = nn.Sequential(
            nn.Linear(16 * 5 * 5, 120), nn.ReLU(), nn.Linear(120, 84), nn.ReLU(), nn.Linear(84, num_classes)
        )

    def forward(self, x):
        return self.classifier(torch.flatten(self.features(x), 1))


class MetaWeightNet(nn.Module):
    """Linear(1,h)-ReLU-Linear(h,1)-sigmoid (reference ``examples/learning_to_reweight/model.py:98-111``;
    the BERT variant scales by 2, ``examples/bert_data_reweighting/model.py:45-59``)."""

    def __init__(self, hidden=100, scale=1.0):
        super().__init__()
        self.fc1 = nn.Linear(1, hidden)
        self.fc2 = nn.Linear(hidden, 1)
        self.scale = scale

    def forward(self, x):
        return torch.sigmoid(self.fc2(F.relu(self.fc1(x)))) * self.scale


def _conv_block(cin, cout):
    # reference ``examples/implicit_maml/models.py:9-24``: conv3x3 -> BN(batch stats) -> ReLU -> pool
    return nn.Sequential(
        nn.Conv2d(cin, cout, 3, stride=1, padding=1, bias=True),
        nn.BatchNorm2d(cout, momentum=1.0, track_running_stats=False),
        nn.ReLU(),
        nn.MaxPool2d(2),
    )


class FourConv(nn.Module):
    """4-conv few-shot backbone (reference ``examples/implicit_maml/models.py:27-119``)."""

    def __init__(self, in_channels, ways, hidden=64, feature_size=64):
        super().__init__()
        self.features = nn.Sequential(
            _conv_block(in_channels, hidden), _conv_block(hidden, hidden),
            _conv_block(hidden, hidden), _conv_block(hidden, hidden),
        )
        self.classifier = nn.Linear(feature_size, ways)

    def forward(self, x):
        f = self.features(x)
        return self.classifier(f.view(f.size(0), -1))


class _ResBlock(nn.Module):
    """CIFAR ResNet basic block with the parameter-free "option A" shortcut and an in-place residual add
    (structure of reference ``examples/learning_to_reweight/model.py:20-52``)."""

    def __init__(self, cin, cout, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, cout, 3, stride=stride, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(cout)
        self.conv2 = nn.Conv2d(cout, cout, 3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(cout)
        self.pad = (cout - cin) // 2 if (stride != 1 or cin != cout) else None

    def forward(self, x):
        out = F.relu(self.bn1(self.conv1(x)))
        out = self.bn2(self.conv2(out))
        sc = x if self.pad is None else F.pad(x[:, :, ::2, ::2], (0, 0, 0, 0, self.pad, self.pad), "constant", 0)
        out += sc
        return F.relu(out)


class ResNetCifar(nn.Module):
    """ResNet-(6n+2) for 32x32 inputs; n=5 is the reference's ResNet32 (``model.py:54-86``)."""

    def __init__(self, n=1, width=16, classes=10):
        super().__init__()
        self.conv1 = nn.Conv2d(3, width, 3, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        blocks, cin = [], width
        for stage, cout in enumerate((width, 2 * width, 4 * width)):
            for b in range(n):
                blocks.append(_ResBlock(cin, cout, 2 if (stage > 0 and b == 0) else 1))
                cin = cout
        self.blocks = nn.Sequential(*blocks)
        self.output = nn.Linear(cin, classes)

    def forward(self, x):
        out = F.relu(self.bn1(self.conv1(x)))
        out = self.blocks(out)
        out = F.avg_pool2d(out, out.size()[3])
        return self.output(out.view(out.size(0), -1))


class MLPNet(nn.Module):
    def __init__(self, din=32, hidden=64, dout=10, depth=2):
        super().__init__()
        layers, d = [], din
        for _ in range(depth):
            layers += [nn.Linear(d, hidden), nn.ReLU()]
            d = hidden
        layers.append(nn.Linear(d, dout))
        self.net = nn.Sequential(*layers)

    def forward(self, x):
        return self.net(x)


# ------------------------------------------------------------------------------------------------
# loss closures (the user-written ``training_step`` bodies)
# ------------------------------------------------------------------------------------------------
def _logistic_lower_step(p: ShimProblem, batch):
    # reference ``test/test_regression.py:47-57``
    inputs, targets = batch
    outs, w = p.module(inputs)
    lam = p.peers["upper"].module()
    return F.binary_cross_entropy_with_logits(outs, targets) + 0.5 * (
        w.unsqueeze(0) @ torch.diag(lam) @ w.unsqueeze(1)
    ).sum()


def _reweighted_ce_step(l2: float):
    # reference ``examples/learning_to_reweight/main.py:117-127`` + explicit L2 (SURVEY §8d)
    def step(p: ShimProblem, batch):
        inputs, labels = batch
        out = p.module(inputs)
        lv = F.cross_entropy(out, labels.long(), reduction="none")
        lv = torch.reshape(lv, (-1, 1))
        weight = p.peers["upper"].module(lv.detach())
        loss = torch.mean(weight * lv)
        if l2 > 0:
            loss = loss + l2 * sum((q ** 2).sum() for q in p.module.parameters())
        return loss

    return step


def _prox_ce_step(reg: float):
    # reference ``examples/implicit_maml/main.py:87-92,122-129``
    def step(p: ShimProblem, batch):
        inputs, labels = batch
        out = p.module(inputs)
        loss = F.cross_entropy(out, labels)
        prox = 0
        for p1, p2 in zip(p.module.parameters(), p.peers["upper"].module.parameters()):
            prox = prox + torch.sum(torch.pow(p1 - p2, 2))
        return loss + reg * prox

    return step


def _roberta_reweight_step(l2: float):
    # reference ``examples/bert_data_reweighting/main.py:117-128``
    def step(p: ShimProblem, batch):
        ids, mask, seg, labels = batch
        logits = p.module(input_ids=ids, attention_mask=mask, token_type_ids=seg).logits
        lv = F.cross_entropy(logits.view(-1, logits.shape[-1]), labels, reduction="none")
        lv = torch.reshape(lv, (-1, 1))
        weight = p.peers["upper"].module(lv.detach())
        loss = torch.mean(weight * lv)
        if l2 > 0:
            loss = loss + l2 * sum((q ** 2).sum() for q in p.module.parameters())
        return loss

    return step


# ------------------------------------------------------------------------------------------------
# factories
# ------------------------------------------------------------------------------------------------
def _pair(name, lower_mod, lower_step, upper_mod, cfg, batch, device, seed_v=1, describe=None):
    lower_mod = lower_mod.to(device)
    upper_mod = upper_mod.to(device)
    lower = ShimProblem("lower", lower_mod, lower_step, cfg)
    upper = ShimProblem("upper", upper_mod, lambda p, b: None, ShimConfig())
    lower.peers["upper"] = upper
    upper.peers["lower"] = lower
    lower.cur_batch = tuple(b.to(device) if torch.is_tensor(b) else b for b in batch)
    g = torch.Generator().manual_seed(seed_v)
    vec = tuple(torch.randn(p.shape, generator=g).to(device) for p in lower_mod.parameters())
    wl = Workload(name, lower, upper, vec, describe or {})
    if cfg.type == "sama":
        # sama preconditions the direction with the lower optimizer's Adam state: make it part of the seeded workload
        with torch.random.fork_rng(devices=[]):
            attach_adam_state(wl)
    return wl


def logistic_hpo(device="cpu", method="neumann", n=500, dim=20, K=5, alpha=1.0, seed=0):
    """Config 1: BCE-with-logits + 0.5*sum(lam_j w_j^2) (reference test/test_regression.py:34-60)."""
    torch.manual_seed(seed)
    x = torch.randn(n, dim)
    w_gt = torch.randn(dim)
    y = ((x @ w_gt + 0.1 * torch.randn(n)) > 0).float()
    lower = LogisticWeights(dim)
    with torch.no_grad():
        lower.w.copy_(0.3 * torch.randn(dim))
    upper = DecayCoefficients(dim)
    with torch.no_grad():
        upper.w.copy_(0.5 + torch.rand(dim))
    cfg = ShimConfig(type=method, neumann_iterations=K, neumann_alpha=alpha, cg_iterations=K, cg_alpha=alpha)
    return _pair("logistic_regression_hpo", lower, _logistic_lower_step, upper, cfg, (x, y), device,
                 describe=dict(n=n, dim=dim, K=K, method=method))


def mlp_reweight(device="cpu", method="cg", batch=64, din=32, hidden=64, classes=10, depth=2, K=5,
                 alpha=1.0, l2=0.05, precision="fp32", seed=0):
    """Small Linear/ReLU/weighted-CE problem used for fast kernel-level parity tests."""
    torch.manual_seed(seed)
    x = torch.randn(batch, din)
    y = torch.randint(0, classes, (batch,))
    lower = MLPNet(din, hidden, classes, depth)
    upper = MetaWeightNet(16)
    cfg = ShimConfig(type=method, precision=precision, neumann_iterations=K, neumann_alpha=alpha, cg_iterations=K,
                     cg_alpha=alpha)
    return _pair("mlp_reweight", lower, _reweighted_ce_step(l2), upper, cfg, (x, y), device,
                 describe=dict(batch=batch, K=K, method=method))


def lenet_reweight(device="cpu", method="cg", batch=100, K=20, alpha=1.0, l2=0.05, seed=0):
    """Config 2: LeNet-5, MWN-weighted CE + 0.05*||w||^2, CG K=20 (SURVEY §8d row 2)."""
    torch.manual_seed(seed)
    x = torch.randn(batch, 3, 32, 32)
    y = torch.randint(0, 10, (batch,))
    lower = LeNet5(10)
    upper = MetaWeightNet(100)
    cfg = ShimConfig(type=method, neumann_iterations=K, neumann_alpha=alpha, cg_iterations=K, cg_alpha=alpha)
    return _pair("learning_to_reweight", lower, _reweighted_ce_step(l2), upper, cfg, (x, y), device,
                 describe=dict(batch=batch, K=K, method=method, model="LeNet-5"))


def resnet_reweight(device="cpu", method="cg", batch=16, n=1, width=16, K=5, alpha=1.0, l2=0.05, seed=0):
    """The reference's own learning_to_reweight model family (ResNet32 = n=5) with the MWN-weighted CE loss."""
    torch.manual_seed(seed)
    x = torch.randn(batch, 3, 32, 32)
    y = torch.randint(0, 10, (batch,))
    lower = ResNetCifar(n, width, 10)
    upper = MetaWeightNet(100)
    cfg = ShimConfig(type=method, neumann_iterations=K, neumann_alpha=alpha, cg_iterations=K, cg_alpha=alpha)
    return _pair("learning_to_reweight_resnet", lower, _reweighted_ce_step(l2), upper, cfg, (x, y), device,
                 describe=dict(batch=batch, n=n, width=width, K=K, method=method))


def fourconv_imaml(device="cpu", method="neumann", n=25, ways=5, image="omniglot", hidden=64, K=20,
                   alpha=0.01, reg=0.5, precision="fp32", seed=0):
    """Config 3: 4-conv backbone, CE + reg*sum||w-theta||^2 (reference examples/implicit_maml/main.py:87-129)."""
    torch.manual_seed(seed)
    if image == "omniglot":
        cin, hw, feat = 1, 28, hidden
    else:
        cin, hw, feat = 3, 84, 5 * 5 * hidden
    x = torch.randn(n, cin, hw, hw)
    y = torch.randint(0, ways, (n,))
    lower = FourConv(cin, ways, hidden, feat)
    upper = FourConv(cin, ways, hidden, feat)
    # theta is a *different* point than w, as after a few inner steps
    with torch.no_grad():
        for pw, pt in zip(lower.parameters(), upper.parameters()):
            pt.copy_(pw + 0.05 * torch.randn_like(pw))
    cfg = ShimConfig(type=method, precision=precision, neumann_iterations=K, neumann_alpha=alpha,
                     cg_iterations=K, cg_alpha=alpha)
    return _pair("implicit_maml", lower, _prox_ce_step(reg), upper, cfg, (x, y), device,
                 describe=dict(n=n, image=image, K=K, method=method, precision=precision))


def roberta_reweight(device="cpu", method="cg", batch=16, seq=50, K=10, alpha=1.0, l2=5e-3, precision="fp32",
                     tiny=False, tiny_hidden=32, seed=0, layers=12):
    """Config 5: HF RobertaForSequenceClassification (random init, eager attention, dropout 0) with
    MWN-weighted CE (reference examples/bert_data_reweighting/main.py:117-128, model.py:11-59).  ``layers`` shortens
    the RoBERTa-base encoder (12 layers) for tests whose float64 reference would not fit in memory at full depth."""
    from transformers import RobertaConfig, RobertaForSequenceClassification

    torch.manual_seed(seed)
    if tiny:
        hc = RobertaConfig(vocab_size=120, hidden_size=tiny_hidden, num_hidden_layers=2, num_attention_heads=4,
                           intermediate_size=2 * tiny_hidden, max_position_embeddings=seq + 4, num_labels=2,
                           hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    else:
        hc = RobertaConfig(vocab_size=50265, hidden_size=768, num_hidden_layers=layers, num_attention_heads=12,
                           intermediate_size=3072, max_position_embeddings=514, type_vocab_size=1,
                           num_labels=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    hc._attn_implementation = "eager"
    lower = RobertaForSequenceClassification(hc)
    lower.train()
    vocab = hc.vocab_size
    ids = torch.randint(3, vocab, (batch, seq))
    mask = torch.ones(batch, seq, dtype=torch.long)
    seg = torch.zeros(batch, seq, dtype=torch.long)
    y = torch.randint(0, 2, (batch,))
    upper = MetaWeightNet(500 if not tiny else 16, scale=2.0)
    cfg = ShimConfig(type=method, precision=precision, neumann_iterations=K, neumann_alpha=alpha,
                     cg_iterations=K, cg_alpha=alpha)
    return _pair("bert_data_reweighting", lower, _roberta_reweight_step(l2), upper, cfg, (ids, mask, seg, y),
                 device, describe=dict(batch=batch, seq=seq, K=K, method=method, precision=precision, tiny=tiny,
                                       **({} if tiny or layers == 12 else dict(layers=layers))))


# -- config 4: a compact DARTS-style supernet (mixed ops weighted by softmax(alpha)) --------------
class _MixedOp(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.ops = nn.ModuleList([
            nn.Identity(),
            nn.Sequential(nn.ReLU(), nn.Conv2d(c, c, 3, padding=1, bias=False), nn.BatchNorm2d(c, affine=False)),
            nn.Sequential(nn.ReLU(), nn.Conv2d(c, c, 3, padding=2, dilation=2, groups=c, bias=False),
                          nn.Conv2d(c, c, 1, bias=False), nn.BatchNorm2d(c, affine=False)),
            nn.AvgPool2d(3, stride=1, padding=1, count_include_pad=False),
        ])

    def forward(self, x, w):
        return sum(wi * op(x) for wi, op in zip(w, self.ops))


class DartsLiteNet(nn.Module):
    """Stem + cells of 2 mixed-op edges each; operation set follows reference
    ``examples/neural_architecture_search/operations.py`` in spirit (skip / conv / dil-sep conv / pool)."""

    def __init__(self, c=16, cells=3, classes=10):
        super().__init__()
        self.stem = nn.Sequential(nn.Conv2d(3, c, 3, padding=1, bias=False), nn.BatchNorm2d(c))
        self.cells = nn.ModuleList([nn.ModuleList([_MixedOp(c), _MixedOp(c)]) for _ in range(cells)])
        self.head = nn.Linear(c, classes)
        self.n_edges = 2 * cells

    def forward(self, x, alphas):
        w = F.softmax(alphas, dim=-1)
        h = self.stem(x)
        e = 0
        for cell in self.cells:
            h = cell[0](h, w[e]) + cell[1](h, w[e + 1])
            e += 2
        return self.head(F.adaptive_avg_pool2d(h, 1).flatten(1))


class ArchParams(nn.Module):
    def __init__(self, n_edges, n_ops=4):
        super().__init__()
        self.alphas = nn.Parameter(1e-3 * torch.randn(n_edges, n_ops))

    def forward(self):
        return self.alphas


def _darts_lower_step(p: ShimProblem, batch):
    # reference ``examples/neural_architecture_search/train_search.py:114-137``
    x, y = batch
    alphas = p.peers["upper"].module()
    return F.cross_entropy(p.module(x, alphas), y)


def _darts_l2_step(l2: float):
    """The DARTS lower loss plus l2*||w||^2: shifts the lower Hessian by 2*l2*I (Neumann / CG parity cases)."""
    if not l2:
        return _darts_lower_step

    def step(p: ShimProblem, batch):
        return _darts_lower_step(p, batch) + l2 * sum((q ** 2).sum() for q in p.module.parameters())

    return step


def _darts_cfg(method, darts_alpha, K, alpha):
    if method == "darts":
        return ShimConfig(type="darts", darts_alpha=darts_alpha)
    return ShimConfig(type=method, darts_alpha=darts_alpha, neumann_iterations=K, neumann_alpha=alpha,
                      cg_iterations=K, cg_alpha=alpha)


def darts_search(device="cpu", batch=16, c=8, cells=2, darts_alpha=0.01, method="darts", K=5, alpha=0.01, l2=0.0,
                 seed=0):
    """Config 4: hypergradient through a DARTS-style supernet -- finite differences (``darts``) or the implicit
    gradient of iDARTS (``neumann`` / ``cg`` with K iterations at step ``alpha``)."""
    torch.manual_seed(seed)
    x = torch.randn(batch, 3, 32, 32)
    y = torch.randint(0, 10, (batch,))
    lower = DartsLiteNet(c, cells, 10)
    upper = ArchParams(lower.n_edges)
    cfg = _darts_cfg(method, darts_alpha, K, alpha)
    describe = dict(batch=batch, c=c, cells=cells, method=method)
    if method != "darts":
        describe.update(K=K, alpha=alpha, l2=l2)
    return _pair("neural_architecture_search", lower, _darts_l2_step(l2), upper, cfg, (x, y), device,
                 describe=describe)



# -- config 4 at full size: the DARTS search network Network(16, 10, 8) + Architecture(4) -------------------------
# Restated from reference ``examples/neural_architecture_search/model_search.py:129-317`` and ``operations.py:5-196``
# (1,930,618 parameters in 1,399 tensors; tests/test_workloads_cpu.py pins the restatement to the reference's own
# classes: same parameter list, same logits).  Under ``darts`` only the finite-difference K4 kernels are ours and the
# two lower forward/backward passes stay on PyTorch (SURVEY.md 8d row 4); under ``neumann`` / ``cg`` the K-loop runs on
# the native plan (depthwise convolutions: csrc/conv_dw.cu).
DARTS_PRIMITIVES = ("none", "max_pool_3x3", "avg_pool_3x3", "skip_connect", "sep_conv_3x3", "sep_conv_5x5",
                    "dil_conv_3x3", "dil_conv_5x5")


def _bn(c, affine=False):
    return nn.BatchNorm2d(c, affine=affine)


def _depthwise_then_pointwise(cin, cout, k, stride, pad, dilation=1):
    return [nn.Conv2d(cin, cin, k, stride=stride, padding=pad, dilation=dilation, groups=cin, bias=False),
            nn.Conv2d(cin, cout, 1, padding=0, bias=False), _bn(cout)]


class _ZeroOp(nn.Module):
    def __init__(self, stride):
        super().__init__()
        self.stride = stride

    def forward(self, x):
        return (x if self.stride == 1 else x[:, :, ::self.stride, ::self.stride]).mul(0.0)


class _HalveResolution(nn.Module):
    """Two stride-2 1x1 convolutions on the even / odd pixel grids, concatenated (operations.py:173-196)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.relu = nn.ReLU()
        self.even = nn.Conv2d(cin, cout // 2, 1, stride=2, bias=False)
        self.odd = nn.Conv2d(cin, cout // 2, 1, stride=2, bias=False)
        self.bn = _bn(cout)

    def forward(self, x):
        x = self.relu(x)
        return self.bn(torch.cat([self.even(x), self.odd(x[:, :, 1:, 1:])], dim=1))


def _darts_op(name, c, stride):
    if name == "none":
        return _ZeroOp(stride)
    if name == "max_pool_3x3":
        return nn.Sequential(nn.MaxPool2d(3, stride=stride, padding=1), _bn(c))
    if name == "avg_pool_3x3":
        return nn.Sequential(nn.AvgPool2d(3, stride=stride, padding=1, count_include_pad=False), _bn(c))
    if name == "skip_connect":
        return nn.Identity() if stride == 1 else _HalveResolution(c, c)
    kind, _, size = name.split("_")
    k = int(size[0])
    if kind == "sep":
        pad = k // 2
        return nn.Sequential(nn.ReLU(), *_depthwise_then_pointwise(c, c, k, stride, pad),
                             nn.ReLU(), *_depthwise_then_pointwise(c, c, k, 1, pad))
    pad = k - 1                                       # dilation 2: "same" padding is (k-1)
    return nn.Sequential(nn.ReLU(), *_depthwise_then_pointwise(c, c, k, stride, pad, dilation=2))


class _MixedEdge(nn.Module):
    def __init__(self, c, stride):
        super().__init__()
        self.ops = nn.ModuleList([_darts_op(name, c, stride) for name in DARTS_PRIMITIVES])

    def forward(self, x, w):
        return sum(wi * op(x) for wi, op in zip(w, self.ops))


class _SearchCell(nn.Module):
    def __init__(self, steps, multiplier, cpp, cp, c, reduction, reduction_prev):
        super().__init__()
        self.reduction, self.steps, self.multiplier = reduction, steps, multiplier
        relu_conv_bn = lambda cin: nn.Sequential(nn.ReLU(), nn.Conv2d(cin, c, 1, bias=False), _bn(c))
        self.pre0 = _HalveResolution(cpp, c) if reduction_prev else relu_conv_bn(cpp)
        self.pre1 = relu_conv_bn(cp)
        self.edges = nn.ModuleList([_MixedEdge(c, 2 if reduction and j < 2 else 1)
                                    for i in range(steps) for j in range(2 + i)])

    def forward(self, s0, s1, weights):
        states = [self.pre0(s0), self.pre1(s1)]
        e = 0
        for _ in range(self.steps):
            states.append(sum(self.edges[e + j](h, weights[e + j]) for j, h in enumerate(states)))
            e += len(states) - 1
        return torch.cat(states[-self.multiplier:], dim=1)


class DartsSearchNetwork(nn.Module):
    """Network(c, classes, layers): stem, `layers` search cells (reduction cells at 1/3 and 2/3), pooled classifier."""

    def __init__(self, c=16, classes=10, layers=8, steps=4, multiplier=4, stem_multiplier=3):
        super().__init__()
        cur = stem_multiplier * c
        self.stem = nn.Sequential(nn.Conv2d(3, cur, 3, padding=1, bias=False), nn.BatchNorm2d(cur))
        cpp, cp, cur = cur, cur, c
        self.cells = nn.ModuleList()
        prev_reduced = False
        for i in range(layers):
            reduced = i in (layers // 3, 2 * layers // 3)
            if reduced:
                cur *= 2
            self.cells.append(_SearchCell(steps, multiplier, cpp, cp, cur, reduced, prev_reduced))
            prev_reduced = reduced
            cpp, cp = cp, multiplier * cur
        self.pool = nn.AdaptiveAvgPool2d(1)
        self.classifier = nn.Linear(cp, classes)

    def forward(self, x, alphas):
        alpha_reduce, alpha_normal = alphas
        s0 = s1 = self.stem(x)
        for cell in self.cells:
            w = F.softmax(alpha_reduce if cell.reduction else alpha_normal, dim=-1)
            s0, s1 = s1, cell(s0, s1, w)
        return self.classifier(self.pool(s1).flatten(1))


class DartsArchitecture(nn.Module):
    """Architecture(steps): alpha_normal / alpha_reduce, one row of 8 op logits per edge (model_search.py:300-317)."""

    def __init__(self, steps=4):
        super().__init__()
        k = sum(2 + i for i in range(steps))
        self.alpha_normal = nn.Parameter(1e-3 * torch.randn(k, len(DARTS_PRIMITIVES)))
        self.alpha_reduce = nn.Parameter(1e-3 * torch.randn(k, len(DARTS_PRIMITIVES)))

    def forward(self):
        return self.alpha_reduce, self.alpha_normal


def darts_search_full(device="cpu", batch=64, c=16, layers=8, darts_alpha=0.01, method="darts", K=5, alpha=0.01,
                      l2=0.0, seed=0):
    """Config 4 as SURVEY.md 8(d) states it: Network(16,10,8) + Architecture(4), x 64x3x32x32 (train_search.py:24).
    ``method`` / ``K`` / ``alpha`` / ``l2`` as in ``darts_search``."""
    torch.manual_seed(seed)
    x = torch.randn(batch, 3, 32, 32)
    y = torch.randint(0, 10, (batch,))
    lower = DartsSearchNetwork(c, 10, layers)
    upper = DartsArchitecture(4)
    cfg = _darts_cfg(method, darts_alpha, K, alpha)
    describe = dict(batch=batch, c=c, layers=layers, method=method)
    if method != "darts":
        describe.update(K=K, alpha=alpha, l2=l2)
    return _pair("neural_architecture_search", lower, _darts_l2_step(l2), upper, cfg, (x, y), device,
                 describe=describe)


def attach_adam_state(wl: Workload, steps: int = 3, lr: float = 1e-2) -> Workload:
    """Give the lower problem an Adam optimizer whose state (exp_avg, exp_avg_sq and the ``last_grad`` the reference's
    ImplicitProblem records, implicit_problem.py:50-66) comes from ``steps`` real Adam steps on the lower loss --
    what ``sama`` preconditions the direction with (reference hypergradient/utils.py:37-63)."""
    opt = torch.optim.Adam(wl.lower.module.parameters(), lr=lr, betas=(0.9, 0.99), eps=1e-8)
    for _ in range(steps):
        opt.zero_grad()
        wl.lower.training_step_exec(wl.lower.cur_batch).backward()
        grads = [p.grad.detach().clone() for p in wl.lower.module.parameters()]
        opt.step()
        for p, g in zip(wl.lower.module.parameters(), grads):
            opt.state[p]["last_grad"] = g
    opt.zero_grad()
    wl.lower.optimizer = opt
    return wl


FACTORIES = {
    "logistic_regression_hpo": logistic_hpo,
    "mlp_reweight": mlp_reweight,
    "learning_to_reweight": lenet_reweight,
    "learning_to_reweight_resnet": resnet_reweight,
    "implicit_maml": fourconv_imaml,
    "neural_architecture_search": darts_search,
    "neural_architecture_search_full": darts_search_full,
    "bert_data_reweighting": roberta_reweight,
}
