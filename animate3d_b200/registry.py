"""threestudio plugin-registry boundary (SURVEY 8b, "threestudio plugin registry").

The reference's guidance / renderer / geometry are threestudio extensions: classes decorated with
`@threestudio.register(name)` (threestudio/__init__.py:5-15), built by `threestudio.find(name)(cfg, ...)`
(threestudio/systems/base.py:292-303, custom/threestudio-animate3d/system/animate3d.py:72) on top of
`BaseObject.__init__(cfg) -> parse_structured(Config, cfg) -> configure(...)` (threestudio/utils/base.py:77-86).

When `threestudio` is importable this module re-exports ITS `register` / `find` / `BaseObject`, so importing
`animate3d_b200.plugins` makes the H100 classes discoverable exactly like the reference's `custom/` directory
(launch.py:70-102).  When it is not (this container, the GPU box), a local registry with the same semantics keeps the
classes constructible and testable; nothing else in the package depends on which of the two is active."""
from __future__ import annotations

import dataclasses
from typing import Any, Dict, Optional

import torch

try:                                                    # the real thing, if the host application has it
    import threestudio as _ts
    from threestudio.utils.base import BaseObject as _TSBaseObject
    HAVE_THREESTUDIO = True
except Exception:                                       # ImportError or any of threestudio's own heavy imports failing
    _ts = None
    _TSBaseObject = None
    HAVE_THREESTUDIO = False

_local_modules: Dict[str, type] = {}


def _modules() -> Dict[str, type]:
    return _ts.__modules__ if HAVE_THREESTUDIO else _local_modules


def register(name: str):
    """threestudio.register: refuses a second class under the same name (threestudio/__init__.py:5-15)."""
    if HAVE_THREESTUDIO:
        return _ts.register(name)

    def decorator(cls):
        if name in _local_modules:
            raise ValueError(f"Module {name} already exists! Names of extensions conflict!")
        _local_modules[name] = cls
        return cls
    return decorator


def find(name: str):
    """threestudio.find incl. the `main:sub1,sub2` mix-in grammar (threestudio/__init__.py:18-31)."""
    if HAVE_THREESTUDIO:
        return _ts.find(name)
    if ":" in name:
        main_name, sub_name = name.split(":")
        names = sub_name.split(",") + [main_name]
        return type(f"{main_name}.{sub_name}", tuple(_local_modules[n] for n in names), {})
    return _local_modules[name]


def parse_structured(fields: Any, cfg: Optional[Any] = None) -> Any:
    """threestudio.utils.config.parse_structured without OmegaConf: unknown keys raise (as OmegaConf.structured does),
    known keys override the dataclass defaults."""
    if cfg is None:
        return fields()
    if dataclasses.is_dataclass(cfg) and not isinstance(cfg, type):
        cfg = dataclasses.asdict(cfg)
    cfg = dict(cfg)
    known = {f.name for f in dataclasses.fields(fields)}
    unknown = [k for k in cfg if k not in known]
    if unknown:
        raise KeyError(f"{fields.__qualname__}: unknown config keys {unknown}")
    return fields(**cfg)


if HAVE_THREESTUDIO:
    BaseObject = _TSBaseObject
else:
    class BaseObject:
        """Local stand-in for threestudio.utils.base.BaseObject (77-86): cfg parsing, `device`, `configure(*args)`."""

        @dataclasses.dataclass
        class Config:
            pass

        cfg: Config

        def __init__(self, cfg: Optional[Any] = None, *args, **kwargs) -> None:
            self.cfg = parse_structured(self.Config, cfg)
            self.device = torch.device("cuda" if torch.cuda.is_available() else "cpu")
            self.configure(*args, **kwargs)

        def configure(self, *args, **kwargs) -> None:
            pass

        # Updateable protocol (threestudio/utils/base.py:14-57): the trainer calls these on every module it owns
        def do_update_step(self, epoch: int, global_step: int, on_load_weights: bool = False):
            self.update_step(epoch, global_step, on_load_weights=on_load_weights)

        def do_update_step_end(self, epoch: int, global_step: int):
            self.update_step_end(epoch, global_step)

        def update_step(self, epoch: int, global_step: int, on_load_weights: bool = False):
            pass

        def update_step_end(self, epoch: int, global_step: int):
            pass


def C(value: Any, epoch: int, global_step: int) -> float:
    """threestudio.utils.misc.C: a scalar, or a [start_step, start_value, end_value, end_step] linear schedule (ints ->
    scheduled by global_step, floats -> by epoch)."""
    if isinstance(value, (int, float)):
        return value
    value = list(value)
    if len(value) == 3:
        value = [0] + value
    if len(value) != 4:
        raise ValueError("Scalar specification only supports list of length 3 or 4, got %d" % len(value))
    start_step, start_value, end_value, end_step = value
    current = global_step if isinstance(end_step, int) else epoch
    return start_value + (end_value - start_value) * max(min(1.0, (current - start_step) / (end_step - start_step)), 0.0)
