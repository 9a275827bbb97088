"""GPU: CUDA-graph execution of the denoiser (mdm_net_set_graph_mode). The first call of a shape signature runs
eagerly, the second is captured, later ones replay; every variant must compute what the eager engine computes on the
same inputs (new inputs every step: staging into the graph's static buffers is part of what is tested)."""
import copy

import pytest
import torch

import parity
import tiny_configs as tc
from mdm_b200 import _lib

pytestmark = pytest.mark.gpu


def _inputs(kind, seed, batch=2):
    nlev = 1 if kind == "unet" else 2
    x, t, lm, mask = tc.seeded_inputs(seed, batch, 16 if nlev == 1 else 32, 6, nlevels=nlev)
    xs = x.cuda() if nlev == 1 else [xi.cuda() for xi in x]
    return xs, t.cuda(), lm.cuda(), mask.cuda()


def _step(model, inp, train):
    xs, t, lm, mask = inp
    if not train:
        with torch.no_grad():
            out = model(xs, t, lm, mask, {})
        return ([o.clone() for o in out] if isinstance(out, list) else [out.clone()]), None
    out = model(xs, t, lm, mask, {})
    outs = list(out) if isinstance(out, list) else [out]
    sum((o * o).sum() for o in outs).backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    return [o.detach().clone() for o in outs], grads


@pytest.mark.parametrize("kind", ["unet", "nested"])
@pytest.mark.parametrize("train", [False, True])
def test_graph_replay_matches_eager(kind, train):
    model, _, _ = parity.tiny_model(tc.TINY[kind])
    eager = copy.deepcopy(model).cuda()
    graph = model.cuda()
    eager.native().set_graph_mode(False)
    graph.native().set_graph_mode(True)
    g0 = _lib.graph_launch_count()
    per_step = []
    for step in range(5):
        inp = _inputs(kind, 100 + step)
        k0 = _lib.launch_count()
        og, gg = _step(graph, inp, train)
        per_step.append(_lib.launch_count() - k0)
        oe, ge = _step(eager, inp, train)
        torch.cuda.synchronize()
        # Not bit-identical even eager vs eager (step 0 here IS eager vs eager and measures 1.0e-3 .. 1.2e-3):
        # GroupNorm partial sums are combined by fp32 atomics, and a 1e-7 change flips fp16 operand roundings
        # downstream. A graph reading stale inputs or dead memory is off by O(1).
        parity.assert_same_run(og, oe, gg, ge)
    # step 0 eager, step 1 captured + launched, steps 2.. replayed: one graph launch per pass
    assert _lib.graph_launch_count() - g0 == (2 if train else 1) * 4
    # the kernels inside the graphs are accounted for: captured and replayed steps report the same number of kernels
    # as each other, and the eager first step that many plus its one-off weight packing launches
    assert len(set(per_step[1:])) == 1 and per_step[1] > 50 and per_step[0] >= per_step[1], per_step


def test_graph_mode_survives_signature_changes_and_weight_updates():
    """Alternating batch sizes (two cached signatures) and an in-place weight update between replays (the fp16
    operand copies are repacked outside the graph, at the addresses the graph reads)."""
    model, _, _ = parity.tiny_model(tc.TINY_UNET)
    eager = copy.deepcopy(model).cuda()
    graph = model.cuda()
    eager.native().set_graph_mode(False)
    for it in range(6):
        inp = _inputs("unet", 200 + it, batch=2 if it % 2 == 0 else 3)
        if it == 4:
            with torch.no_grad():
                for pa, pb in zip(graph.parameters(), eager.parameters()):
                    pa.mul_(1.01)
                    pb.mul_(1.01)
        og, _ = _step(graph, inp, False)
        oe, _ = _step(eager, inp, False)
        parity.assert_same_run(og[:1], oe[:1])
