"""``modal.App``: registry + decorators.  ``@app.function`` / ``@app.cls`` / ``@app.local_entrypoint`` with the
keyword census of SURVEY.md §2.2; unknown keywords are accepted and recorded (cloud-only knobs have no in-box
meaning), ``gpu=`` is parsed to a local H100 count."""
from __future__ import annotations

import contextlib
import inspect
import json
import os
import sys

from . import _runtime as rt
from .cls import Cls, marks
from .functions import Function
from .gpu import parse_gpu_count

_apps: dict[str, "App"] = {}


def _registry_path():
    from .resources import state_dir

    return os.path.join(state_dir(), "deployed.json")


def _read_registry() -> dict:
    try:
        with open(_registry_path()) as f:
            return json.load(f)
    except (OSError, ValueError):
        return {}


def _lookup_app(name):
    """An app of this process, else one that `modal deploy` recorded from another process (`modal deploy x.py` followed by
    `modal.Cls.from_name(app_name, ...)` in a client script: 06_gpu_and_ml/gpu_snapshot.py:64-77): its file is imported here."""
    if name in _apps:
        return _apps[name]
    ent = _read_registry().get(name)
    if ent and os.path.exists(ent.get("path", "")):
        import importlib.util

        mod_name = "_modal_deployed_" + "".join(c if c.isalnum() else "_" for c in name)
        spec = importlib.util.spec_from_file_location(mod_name, ent["path"])
        mod = importlib.util.module_from_spec(spec)
        sys.modules[mod_name] = mod
        sys.path.insert(0, os.path.dirname(ent["path"]))
        spec.loader.exec_module(mod)
    return _apps.get(name)


class LocalEntrypoint:
    def __init__(self, raw_f, app):
        self.raw_f, self.app = raw_f, app
        self.__name__ = raw_f.__name__
        self.__doc__ = raw_f.__doc__

    def __call__(self, *a, **k):
        with self.app.run():
            out = self.raw_f(*a, **k)
            if inspect.isawaitable(out):
                return rt.run_maybe_async(lambda: out)
            return out


class App:
    def __init__(self, name=None, *, image=None, secrets=None, volumes=None, **kwargs):
        self.name = name
        self.description = name
        self.image, self.secrets, self.volumes = image, list(secrets or []), dict(volumes or {})
        self.registered_functions: dict[str, Function] = {}
        self.registered_classes: dict[str, Cls] = {}
        self.registered_entrypoints: dict[str, LocalEntrypoint] = {}
        self.registered_web_endpoints: list[str] = []
        self.app_id = rt.new_object_id("ap")
        self._running = 0
        if name:
            _apps[name] = self

    # ---- decorators
    def _options(self, kw):
        o = dict(kw)
        o.setdefault("image", self.image)
        o["gpu_count"] = parse_gpu_count(o.get("gpu"))
        vols = dict(self.volumes)
        vols.update(o.get("volumes") or {})
        o["volumes"] = vols
        for path, vol in vols.items():
            if hasattr(vol, "mount_at"):
                vol.mount_at(path)
        return o

    def function(self, _fn=None, **kwargs):
        def deco(fn):
            if isinstance(fn, Function):
                fn.options.update(self._options(kwargs))
                return fn
            opts = self._options(kwargs)
            m = marks(fn)
            if "max_inputs" in m:
                opts["max_inputs"] = m["max_inputs"]
            batcher = None
            if "batched" in m:
                holder = {}

                def batcher():
                    if "b" not in holder:
                        holder["b"] = rt.Batcher(fn, m["batched"][0], m["batched"][1])
                    return holder["b"]
            f = Function(fn, tag=kwargs.get("name") or fn.__name__, app=self, options=opts, batcher=batcher)
            self.registered_functions[f.tag] = f
            if "web" in m:
                self.registered_web_endpoints.append(f.tag)
            return f

        return deco(_fn) if callable(_fn) else deco

    def cls(self, _cls=None, **kwargs):
        def deco(user_cls):
            c = Cls(user_cls, self, self._options(kwargs))
            self.registered_classes[user_cls.__name__] = c
            return c

        return deco(_cls) if inspect.isclass(_cls) else deco

    def local_entrypoint(self, _fn=None, **kwargs):
        def deco(fn):
            e = LocalEntrypoint(fn, self)
            self.registered_entrypoints[fn.__name__] = e
            return e

        return deco(_fn) if callable(_fn) else deco

    # ---- lifecycle
    @contextlib.contextmanager
    def run(self, **_kw):
        self._running += 1
        try:
            yield self
        finally:
            self._running -= 1
            if self._running == 0:
                from .cls import _shutdown_all

                _shutdown_all()

    def deploy(self, *, _source=None, **_kw):
        """In-process registration plus a record under the state directory so that another process's `from_name` /
        `lookup` finds the app (the deployed app's code is its source file, re-imported there)."""
        if self.name:
            _apps[self.name] = self
            src = _source
            if src is None:
                f = sys._getframe(1)
                src = f.f_globals.get("__file__")
            if src:
                reg = _read_registry()
                reg[self.name] = {"path": os.path.abspath(src)}
                os.makedirs(os.path.dirname(_registry_path()), exist_ok=True)
                tmp = _registry_path() + f".{os.getpid()}.tmp"
                with open(tmp, "w") as f:
                    json.dump(reg, f, indent=1)
                os.replace(tmp, _registry_path())
        return self

    def include(self, other: "App"):
        self.registered_functions.update(other.registered_functions)
        self.registered_classes.update(other.registered_classes)
        return self

    @staticmethod
    def lookup(name, *, create_if_missing=False, **_kw) -> "App":
        if name in _apps:
            return _apps[name]
        if create_if_missing:
            return App(name)
        from .exception import NotFoundError

        raise NotFoundError(f"App {name!r} not found in this process")

    def __repr__(self):
        return f"<modal.App {self.name!r}>"


Stub = App  # legacy alias still present in the tree (SURVEY.md §2.2)


@contextlib.contextmanager
def enable_output(*_a, **_k):
    yield
