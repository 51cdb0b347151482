"""The synthetic workloads restate the reference examples' models (betty_b200/workloads.py cites each); this pins the
config-4 restatement -- Network(16, 10, 8) + Architecture(4) -- to the reference's own classes: identical parameter list
and identical logits on the same weights (tests/golden/models/darts_network.pt, made by oracle/make_golden.py from the
reference's examples/neural_architecture_search/model_search.py)."""
import os

import torch

from betty_b200 import workloads as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "models", "darts_network.pt")


def test_full_size_darts_network_has_the_survey_sizes():
    net, arch = W.DartsSearchNetwork(16, 10, 8), W.DartsArchitecture(4)
    ps = list(net.parameters())
    assert sum(p.numel() for p in ps) == 1_930_618 and len(ps) == 1_399       # SURVEY.md 8(a)
    assert sum(p.numel() for p in arch.parameters()) == 2 * 14 * 8


def test_full_size_darts_network_matches_the_reference_classes():
    rec = torch.load(GOLDEN, weights_only=False)
    torch.manual_seed(0)
    net, arch = W.DartsSearchNetwork(16, 10, 8), W.DartsArchitecture(4)
    assert [tuple(p.shape) for p in net.parameters()] == [tuple(s) for s in rec["shapes"]]
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(1))
    net.train()
    with torch.no_grad():
        assert torch.allclose(net(x, arch()), rec["logits"], rtol=1e-5, atol=1e-6)
