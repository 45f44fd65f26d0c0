"""Host logic of CUDA-graph capture (animate3d_b200/capture.py, rasterizer / renderer / mesh capture paths): the captured
pair capacity and its growth after an overflow, the step / capture / retry policy of StepGraphs, the camera -> timestamp
layout, and the (seed, offset) state of the captured mesh-edge sampler against the oracle's Philox draw."""
import numpy as np
import pytest
import torch

from animate3d_b200 import rasterizer as RZ
from animate3d_b200.capture import MAX_RETRIES, StepGraphs
from animate3d_b200.mesh import MeshGraph
from animate3d_b200.renderer import _device_index, timestamp_layout
from oracle import mesh_oracle as MO


def test_capacity_and_growth():
    key = ("cpu-test", 256, 256, 60)
    RZ._cap_hint.pop(key, None)
    assert RZ.capture_capacity(100000) == int(100000 * RZ.CAPTURE_SLACK) > 100000
    grown = RZ.grow_hint(key, 500000)
    assert grown == int(500000 * 1.08) + 1024 and RZ._cap_hint[key] == grown
    assert RZ.capture_capacity(grown) > 500000                       # the recapture holds what the replay needed
    assert RZ.grow_hint(key, 10) == grown                            # never shrinks
    RZ._cap_hint.pop(key)


class _Opt:
    def __init__(self, fused=True, capturable=True):
        self.param_groups = [{"fused": fused, "capturable": capturable, "params": []}]


class _Policy(StepGraphs):
    """StepGraphs with its device work replaced by a log; `overflows` replays report an overflow."""

    def __init__(self, overflows=0):
        super().__init__(lambda inp: None, _Opt())
        self.log, self.overflows = [], overflows

    def eager(self, inputs):
        self.log.append("eager")

    def capture(self, key, inputs):
        self.log.append(("capture", key))
        self.graphs[key] = None

    def replay(self, key, inputs):
        self.log.append(("replay", key))
        if self.overflows:
            self.overflows -= 1
            return True
        return False


def test_step_policy():
    p = _Policy()
    assert p.step("a", {}) is False and p.log == ["eager"]          # first step of a layout: eager warm-up
    assert p.step("a", {}) is True and p.log[1:] == [("capture", "a"), ("replay", "a")]
    assert p.step("a", {}) is True and p.log[3:] == [("replay", "a")]
    assert p.step("b", {}) is False and p.step("b", {}) is True     # a second layout gets its own graph
    assert p.step("a", {}) is True and p.log[-1] == ("replay", "a")


def test_overflow_recaptures_and_reruns():
    p = _Policy(overflows=1)
    p.step("a", {})
    assert p.step("a", {}) is True
    assert p.log[1:] == [("capture", "a"), ("replay", "a"), ("capture", "a"), ("replay", "a")] and p.recaptures == 1
    q = _Policy(overflows=MAX_RETRIES)
    q.step("a", {})
    with pytest.raises(RuntimeError, match="still overflowed"):
        q.step("a", {})


def test_needs_fused_capturable_adam():
    for opt in (_Opt(fused=False), _Opt(capturable=False)):
        with pytest.raises(ValueError, match="fused=True, capturable=True"):
            StepGraphs(lambda inp: None, opt)


@pytest.mark.parametrize("ts", [np.tile(np.linspace(-1, 1, 16)[1:5], 4), np.tile(np.linspace(-1, 1, 16)[[3, 15]], 4),
                                np.array([0.5, -0.25, 0.5, 0.1, -0.25])])
def test_timestamp_layout_is_unique_inverse(ts):
    layout = timestamp_layout(ts)
    _, inv = torch.unique(torch.tensor(ts, dtype=torch.float32), return_inverse=True)
    assert list(layout) == inv.tolist()
    assert torch.equal(_device_index(layout, "cpu"), inv)


def test_mesh_sample_state_matches_oracle_offsets():
    """Replay k of a captured sample(K) uses (seed, offset0 + k): the state holds them as the kernel reads them (uint64
    words), and consecutive offsets give the oracle's distinct tables."""
    verts, _, polys, _ = MO.fixture_mesh(seed=1)
    faces = np.asarray([[p[0][0], p[k][0], p[k + 1][0]] for p in polys for k in range(1, len(p) - 1)], np.int64)
    row_ptr, col = MO.csr_from_faces(faces, verts.shape[0])
    g = MeshGraph(torch.from_numpy(np.asarray(row_ptr, np.int32)), torch.from_numpy(np.asarray(col, np.int32)))
    seed, offset0 = (1 << 62) + 12345, (1 << 33) + 7
    g.set_sample_state(seed, offset0)
    assert g.sample_state.dtype == torch.int64 and g.sample_offset() == offset0
    words = g.sample_state.numpy().view(np.uint64)
    assert int(words[0]) == seed and int(words[1]) == offset0
    tables = [MO.sample_csr(row_ptr, col, 3, int(words[0]), int(words[1]) + k) for k in range(3)]
    assert not np.array_equal(tables[0], tables[1]) and not np.array_equal(tables[1], tables[2])
    for bad in ((-1, 0), (0, 1 << 63)):
        with pytest.raises(ValueError):
            g.set_sample_state(*bad)
