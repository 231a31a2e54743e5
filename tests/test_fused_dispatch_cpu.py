"""CPU tests of fused.fused_forward / fused.train_forward's dispatch by class name: the reference classes with no custom
layer (FlowNet2S, FlowNet2SD) have no fused data flow and are refused before anything touches a tensor, and the error
names every class that has one."""
import pytest
import torch


def _net(name):
    return type(name, (torch.nn.Module,), {})()


@pytest.mark.parametrize("name", ["FlowNet2S", "FlowNet2SD"])
def test_networks_without_custom_layers_are_refused(name):
    from flownet2_b200 import fused
    x = torch.zeros(1, 3, 2, 8, 8)
    with pytest.raises(TypeError, match="no fused data flow for %s \\(FlowNet2, FlowNet2CSS, FlowNet2CS, FlowNet2C, "
                                        "FlowNetC\\)" % name):
        fused.fused_forward(_net(name), x)
    with pytest.raises(TypeError, match="no fused data flow for %s \\(FlowNet2CSS, FlowNet2CS, FlowNet2C, FlowNetC\\)"
                                        % name):
        fused.train_forward(_net(name), x)
