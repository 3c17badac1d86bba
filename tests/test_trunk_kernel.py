"""The conditioner trunk as ONE launch: the coupling-step kernel stopped after its last trunk layer (`h_hi / h_lo` of
NfkCouplingStep, `trunk_step` in the timeline) -- what dense.run_trunk uses for every plain ResidualNet / MLP trunk whose last
layer is NOT fused with a spline (affine couplings, unfused routes).  Host planning is tested on the CPU, the kernel on a GPU."""
import pytest
import torch

from conftest import rel_err
from nflows_b200 import config
from nflows_b200 import dense as D
from nflows_b200 import kernels as K
from nflows_b200.nn.nets import MLP, ResidualNet


def test_plan_follows_the_residual_block_structure():
    net = ResidualNet(24, 48, hidden_features=64, num_blocks=2).eval()
    flags = D.plan_step_kernel(net.dense_chain(None))
    # initial layer: its fp32 output is the first block's skip tensor (4) and the block's first layer takes relu of it (8);
    # block = [relu -> W -> relu] [W + skip]; the first block's output is the second block's skip tensor
    assert flags == [4 | 8, 1, 2 | 4 | 8, 1, 2]
    mlp = MLP([24], [48], [64, 64, 64, 64]).eval()
    assert D.plan_step_kernel(mlp.dense_chain(None)) == [1, 1, 1, 1]      # relu outputs, no skips, consumers take them as they are
    net.blocks[0].use_batch_norm = True
    assert net.dense_chain(None) is None                                  # not a plain relu trunk: torch path


@pytest.mark.gpu
@torch.no_grad()
@pytest.mark.parametrize("hidden,blocks,rows", [(256, 2, 1000), (64, 1, 130), (128, 3, 4096),
                                                # two 128-column chunks, the second 32, 64 and 96 wide; 8 square layers
                                                (160, 4, 129), (192, 4, 4096), (224, 4, 1000)])
def test_trunk_step_matches_the_layer_by_layer_path(cuda_device, hidden, blocks, rows):
    torch.manual_seed(hidden + blocks)
    net = ResidualNet(40, 16, hidden_features=hidden, num_blocks=blocks).eval()
    for p in net.parameters():
        p.add_(torch.randn_like(p) * 0.05)
    x = torch.randn(rows, 40)
    # fp64 value of the trunk output (input of the final layer)
    h = net.double().initial_layer(x.double())
    for block in net.blocks:
        h = block(h)
    net = net.float().to(cuda_device)
    chain = net.dense_chain(None)
    xd = x.to(cuda_device)
    K.TIMELINE = []
    try:
        got = D.run_trunk(chain, xd, None, True).pair.float().cpu()
        tags = [t[0] for t in K.TIMELINE]
    finally:
        K.TIMELINE = None
    assert any(t.startswith("trunk_step") for t in tags) and not any(t.startswith("linear_") for t in tags), tags
    config.coupling_step_kernel = False
    try:
        base = D.run_trunk(chain, xd, None, True).pair.float().cpu()
    finally:
        config.coupling_step_kernel = True
    assert rel_err(got, h) <= 1e-5 and rel_err(base, h) <= 1e-5
    assert rel_err(got, base) <= 5e-6
