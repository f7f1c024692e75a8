"""CPU: the resumable LM loop behind background pose-graph optimisation (pose_graph._LMState), and the replay entry.

_LMState is driven on scripted step results, (candidate, loss before, loss after, Cholesky ok) per active graph, and
must make the decisions of the loop it replaced (the transcription below): the same steps requested with the same
dampings, the same candidates accepted, the same loss histories and the same graphs leaving at the same iteration."""
import random

import pytest

from vista_slam_b200 import pose_graph as P


def _reference_iterations(graphs, step, steps, patience, decreasing, radius):
    """The LM loop of slam.py:121-134 as pose_graph._lm_iterations ran it before it became a state machine."""
    n = len(graphs)
    radii, stall, losses = [radius] * n, [0] * n, [[] for _ in range(n)]
    active = list(range(n))
    for _ in range(steps):
        if not active:
            break
        results = step(active, [1.0 / radii[k] for k in active])
        still = []
        for k, (cand, l0, l1, ok) in zip(active, results):
            if ok and l1 <= l0:
                graphs[k].nodes = cand
                radii[k] = min(radii[k] * 2.0, 1e32)
            else:
                radii[k] = max(radii[k] * 0.5, 1e-32)
                l1 = l0
            losses[k].append(l1)
            stall[k] = stall[k] + 1 if (l0 - l1) < decreasing else 0
            if stall[k] < patience:
                still.append(k)
        active = still
    return losses


class _Graph:
    def __init__(self):
        self.nodes, self.history = None, []

    def __setattr__(self, k, v):
        if k == "nodes" and v is not None:
            self.history.append(v)
        object.__setattr__(self, k, v)


def _script(seed, kinds):
    """step(active, dampings) answering from a per-graph script: kinds[k] lists what graph k's successive steps do."""
    rng = random.Random(seed)
    calls, loss, count = [], {}, {}

    def step(active, dampings):
        calls.append((list(active), list(dampings)))
        out = []
        for k in active:
            c = count.get(k, 0)
            count[k] = c + 1
            kind = kinds[k][min(c, len(kinds[k]) - 1)]
            l0 = loss.setdefault(k, 10.0 + rng.random())
            if kind == "good":  # a decrease well above `decreasing`
                l1, ok = l0 * rng.uniform(0.3, 0.9), True
            elif kind == "flat":  # a decrease below `decreasing`: counts towards the plateau
                l1, ok = l0 - rng.uniform(0.0, 5e-5), True
            elif kind == "worse":  # rejected: the loss went up
                l1, ok = l0 * rng.uniform(1.01, 2.0), True
            elif kind == "chol":  # rejected: the Cholesky failed, whatever the losses say
                l1, ok = l0 * 0.5, False
            else:
                raise AssertionError(kind)
            if ok and l1 <= l0:
                loss[k] = l1
            out.append((("cand", k, c), l0, l1, ok))
        return out

    return step, calls


CASES = {
    "accept_all": [["good"]],
    "rejected": [["good", "worse", "good", "worse", "worse", "good"]],
    "cholesky": [["chol", "good", "chol", "chol", "good"]],
    "plateau": [["good", "flat", "flat", "flat", "good"]],
    "plateau_reset": [["flat", "flat", "good", "flat", "flat", "good", "flat", "flat", "flat"]],
    "rejections_plateau": [["worse", "worse", "worse", "good"]],
    "group_stops_apart": [["good", "flat", "flat", "flat"], ["good"], ["chol", "chol", "chol"],
                          ["good", "good", "worse", "flat", "chol", "flat"], ["flat", "good", "flat", "flat", "flat"]],
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("steps", [0, 1, 4, 20])
def test_state_machine_reproduces_the_loop(case, steps):
    kinds = CASES[case]
    kw = dict(steps=steps, patience=3, decreasing=1e-4, radius=1e4)
    ref_graphs, got_graphs, drv_graphs = ([_Graph() for _ in kinds] for _ in range(3))
    step, ref_calls = _script(5, kinds)
    want = _reference_iterations(ref_graphs, step, **kw)
    step, calls = _script(5, kinds)
    assert P._lm_iterations(got_graphs, step, **kw) == want
    assert calls == ref_calls
    # driven one step at a time, as PoseGraphRun.poll does
    step, drv_calls = _script(5, kinds)
    state = P._LMState(len(kinds), kw["steps"], kw["patience"], kw["decreasing"], kw["radius"])
    while not state.done:
        active, damp = list(state.active), state.dampings()
        state.advance(drv_graphs, step(active, damp))
    assert state.losses == want and drv_calls == ref_calls
    assert state.iterations == len(ref_calls) <= steps
    for a, b, c in zip(ref_graphs, got_graphs, drv_graphs):
        assert a.history == b.history == c.history
    if steps == 20 and case == "group_stops_apart":
        # members leave at different iterations, and the plateau stops the group before 20 steps
        assert len({len(h) for h in want}) > 2 and len(ref_calls) < 20
    if steps == 20 and case in ("rejected", "cholesky"):
        assert any(d[0] > 1e-4 for _, d in ref_calls[1:])  # a rejection grew the damping


def test_replay_entry_is_declared_and_refuses_a_null_graph():
    from vista_slam_b200 import _lib
    L = _lib.lib()
    assert hasattr(L, "sta_graph_replay_nodes")
    with open(_lib.os.path.join(_lib._HERE, "..", "include", "sta_b200.h")) as f:
        assert "int sta_graph_replay_nodes(StaGraph* g, int count, const int* triples_host, void* stream);" in f.read()
    assert L.sta_graph_replay_nodes(None, 0, None, None) != 0
    assert b"null graph" in L.sta_last_error()
