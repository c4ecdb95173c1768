"""Host side of the layout operators' autograd routing, without a GPU: the SVG1 paths that have no backward raise
SvgbError under grad before any device work (the inputs here are CPU tensors, so any device work would fail first,
with another message), and without grad they are unchanged."""
import pytest
import torch


def _inputs(requires_grad):
    return [torch.zeros(1, 2, 64 + 2 * 128, 128, dtype=torch.bfloat16, requires_grad=requires_grad) for _ in range(3)]


def _calls():
    from svgb200.models import common

    core = common.SVG1Core(64, 2, 128)
    fp8 = common.SVG1Core(64, 2, 128, fp8=True)
    return {
        "fp8": lambda q, k, v: fp8.sparse_core(q, k, v),
        "head-parallel": lambda q, k, v: core.sparse_core_head_parallel(q, k, v, None),
        "host-pipelined": lambda q, k, v: core.sparse_core_from_host(q, k, v, torch.empty_like(q)),
    }


@pytest.mark.parametrize("path", ["fp8", "head-parallel", "host-pipelined"])
def test_svg1_paths_without_backward_raise_under_grad(path):
    from svgb200 import core

    with pytest.raises(core.SvgbError, match=f"{path}.*has no backward"):
        _calls()[path](*_inputs(True))


@pytest.mark.parametrize("path", ["fp8", "head-parallel", "host-pipelined"])
def test_svg1_paths_without_grad_are_unchanged(path):
    """Without grad (torch.no_grad, or inputs that do not require grad) the entry check passes and the call proceeds
    to its first device work, which needs CUDA tensors."""
    from svgb200 import core

    for grad, ctx in ((True, torch.no_grad), (False, torch.enable_grad)):
        with ctx(), pytest.raises((core.SvgbError, AttributeError)) as e:
            _calls()[path](*_inputs(grad))
        assert "no backward" not in str(e.value)


def test_layout_ops_route_on_needs_grad():
    """head_placement and the permutations reject CPU tensors with or without grad: the autograd Functions are reached
    only after the same argument checks as the plain calls."""
    from svgb200 import core

    x = _inputs(True)
    outs = [torch.zeros_like(t) for t in x]
    best = torch.zeros(1, 2, dtype=torch.long)
    perm = torch.arange(x[0].shape[2]).expand(2, -1)
    for grad in (True, False):
        with torch.set_grad_enabled(grad):
            with pytest.raises(core.SvgbError, match="CUDA"):
                core.head_placement(x, outs, best, 64, 2, 128)
            with pytest.raises(core.SvgbError, match="CUDA"):
                core.permute_gather(x[0], perm)
            with pytest.raises(core.SvgbError, match="CUDA"):
                core.permute_scatter(x[0], perm)
