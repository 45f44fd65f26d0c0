"""Replay the body of a motion-reconstruction or mesh-animation `training_step` (systems/animate3d.py:120-244: deform ->
batched render -> rgb / mask MSE -> ARAP -> backward -> Adam) from CUDA graphs.

`StepGraphs(step_fn, optimizer)` keeps one graph per layout key, all in one memory pool.  A layout is whatever fixes the
shapes and the host-side choices of a step: for the "normal" sampling strategy the `start_index` (the number of frames and
the camera -> timestamp map), for "light" the fixed 2 frames x 4 views.  The values that change from step to step --
timestamps, camera rows, targets -- are tensors in `inputs`; `step(key, inputs)` copies them into the layout's static
buffers and replays.  The graph draws its own randomness on the device: the 10 % gradient mask and the ARAP node sample
from torch's CUDA generator, the mesh-edge neighbours from the MeshGraph's device state (`MeshGraph.set_sample_state`).

The first step of a layout runs eagerly: it is a real training step, and it sizes the rasterizer's captured pair capacity
(`rasterizer.capture_capacity`).  A replay whose render needed more pairs than that sets a device flag that the fused Adam
kernel reads as `found_inf`, so the parameters and the optimizer state stay exactly as they were; `step` reads that flag
once per step, grows the capacity, captures again and re-runs the step.

Tensors a graph leaves alive (the outputs `step_fn` keeps, `arap.last_sample_idx`) hold the values of that graph's last
replay until another graph of the same pool replays.

The engine networks a refine step calls (the UNet, the CLIP tower, the VAE) keep persistent buffers and packed weights that
a graph records by address.  Each keeps a counter, `capture_version`, that it bumps whenever one of those tensors may have
moved (buffer growth, `load_state_dict`, `.to()`, repacking).  Recorded under a capture, such a module registers itself and
its counter (`note_module`); before each replay `step` compares the counters and captures again on any change, so a replay
never runs on freed or stale memory.  These recaptures are counted in `pointer_recaptures`, overflow ones in `recaptures`."""
from __future__ import annotations

import contextlib
from typing import Callable, Dict, Hashable, List, Optional, Tuple

import torch

from . import rasterizer

MAX_RETRIES = 3
_module_log: Optional[list] = None


@contextlib.contextmanager
def collect_modules():
    """Modules recorded inside this context (through `note_module`) append (module, its capture_version) to the yielded
    list, once each."""
    global _module_log
    prev, _module_log = _module_log, []
    try:
        yield _module_log
    finally:
        _module_log = prev


def capturing(device) -> bool:
    """Whether the current stream of `device` is being captured into a CUDA graph (False for a CPU device, where the query
    itself would need a driver)."""
    return torch.device(device).type == "cuda" and torch.cuda.is_current_stream_capturing()


def note_module(module) -> None:
    """Called by a module whose kernels are being recorded into a graph: the graph depends on its buffers and weights staying
    where they are, which `module.capture_version` tracks."""
    if _module_log is not None and all(m is not module for m, _ in _module_log):
        _module_log.append((module, module.capture_version))


class StepGraphs:
    """step_fn(inputs) runs the forward and backward of one step on the tensors of `inputs`, leaving the gradients in .grad
    (it does not zero them or step the optimizer).  optimizer: torch.optim.Adam(..., fused=True), the only Adam whose kernel
    honours `found_inf`, created with capturable=True; a learning-rate schedule needs tensor learning rates, updated in
    place before each step."""

    def __init__(self, step_fn: Callable[[Dict[str, torch.Tensor]], None], optimizer: torch.optim.Optimizer):
        if not all(g.get("fused") and g.get("capturable") for g in optimizer.param_groups):
            raise ValueError("StepGraphs needs torch.optim.Adam(..., fused=True, capturable=True): only the fused kernel skips "
                             "an update on the found_inf flag that gates an overflowed render")
        self.step_fn, self.optimizer = step_fn, optimizer
        self.graphs: Dict[Hashable, tuple] = {}        # key -> (CUDAGraph, [(raster key, device [pairs, overflow])])
        self.static: Dict[Hashable, Dict[str, torch.Tensor]] = {}
        self.warm = set()
        self.modules: Dict[Hashable, List[Tuple[object, int]]] = {}     # key -> the modules its graph recorded, and their versions
        self.recaptures = 0             # after an overflowed replay
        self.pointer_recaptures = 0     # after a recorded module's buffers or weights moved
        self.pool = None
        self.found_inf = None

    def step(self, key: Hashable, inputs: Dict[str, torch.Tensor]) -> bool:
        """One training step of layout `key`.  Returns False when it ran eagerly (the first step of a layout), True when it
        ran from the graph."""
        if key not in self.warm:
            self.eager(inputs)
            self.warm.add(key)
            return False
        if key not in self.graphs:
            self.capture(key, inputs)
        elif self.stale(key):
            self.capture(key, inputs)
            self.pointer_recaptures += 1
        for _ in range(MAX_RETRIES):
            if not self.replay(key, inputs):
                return True
            self.capture(key, inputs)
            self.recaptures += 1
        raise RuntimeError(f"layout {key!r}: the render still overflowed after {MAX_RETRIES} larger captures")

    def release(self) -> None:
        """Drop every graph and the memory pool they share; the next step of each layout captures again (no eager first
        step).  A process that alternates with large eager work can hand the pool's memory back this way."""
        self.graphs.clear()
        self.modules.clear()
        self.pool = None

    def stale(self, key: Hashable) -> bool:
        """Whether a module the graph of `key` recorded has bumped its capture_version since."""
        return any(m.capture_version != v for m, v in self.modules.get(key, ()))

    def eager(self, inputs: Dict[str, torch.Tensor]) -> None:
        """The step without a graph."""
        self.optimizer.zero_grad(set_to_none=True)
        self.step_fn(inputs)
        self.optimizer.step()

    def _copy_in(self, key, inputs):
        st = self.static.get(key)
        if st is None:
            st = self.static[key] = {k: v.clone() for k, v in inputs.items()}
        else:
            for k, v in inputs.items():
                st[k].copy_(v)
        return st

    def capture(self, key: Hashable, inputs: Dict[str, torch.Tensor]) -> None:
        """(Re)capture the step of `key`.  The capture runs no kernel: parameters are untouched until `replay`."""
        dev = self.optimizer.param_groups[0]["params"][0].device
        if self.pool is None:
            self.pool = torch.cuda.graph_pool_handle()
            self.found_inf = torch.zeros((), device=dev)      # 0-dim, like the Adam step counters it is subtracted from
        st = self._copy_in(key, inputs)
        # a graph being replaced stays alive until the new one is captured: the pool is released with its last graph
        self.optimizer.zero_grad(set_to_none=True)      # the graph allocates its own gradients
        g = torch.cuda.CUDAGraph()
        self.optimizer.found_inf = self.found_inf
        try:
            with rasterizer.collect_pair_counts() as log, collect_modules() as mods, torch.cuda.graph(g, pool=self.pool):
                self.step_fn(st)
                if log:
                    self.found_inf.copy_(torch.stack([c[1] for _, c in log]).amax())
                else:
                    self.found_inf.zero_()
                self.optimizer.step()
        finally:
            del self.optimizer.found_inf
        self.graphs[key] = (g, list(log))
        self.modules[key] = list(mods)

    def replay(self, key: Hashable, inputs: Dict[str, torch.Tensor]) -> bool:
        """Copy `inputs` into the static buffers of `key` and replay its graph.  Returns True when a render overflowed: the
        update was skipped and the capacity hint of that render has been grown (the caller captures again)."""
        g, log = self.graphs[key]
        self._copy_in(key, inputs)
        g.replay()
        if not bool(self.found_inf.item()):             # the one host read of a step
            return False
        for rkey, counts in log:
            needed, overflowed = (int(x) for x in counts.tolist())
            if overflowed:
                rasterizer.grow_hint(rkey, needed)
        return True
