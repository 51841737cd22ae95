"""Volume / Secret / Dict / Queue / schedules / retries: the non-compute objects scripts construct at import
time.  Volumes map to local directories under ``$MODAL_SHIM_STATE`` (default ``~/.modal_b200``); absolute mount
points such as ``/data`` (text_embeddings_inference.py:27,144) resolve into them through virtual mounts
(``_mounts.py``) -- the runtime does not touch paths outside its state dir (``MODAL_SHIM_MOUNTS=link`` symlinks instead).  Dict and
Queue are in-process (09_job_queues is OUT OF SCOPE, this is the minimum for scripts to import and run locally)."""
from __future__ import annotations

import collections
import os
import queue as _queue
import shutil
import threading
from dataclasses import dataclass

from .exception import NotFoundError


def state_dir() -> str:
    d = os.environ.get("MODAL_SHIM_STATE") or os.path.join(os.path.expanduser("~"), ".modal_b200")
    os.makedirs(d, exist_ok=True)
    return d


class Volume:
    _named: dict[str, "Volume"] = {}

    def __init__(self, name: str):
        self.name = name
        self.object_id = f"vo-{name}"

    @property
    def local_path(self) -> str:
        p = os.path.join(state_dir(), "volumes", self.name)
        os.makedirs(p, exist_ok=True)
        return p

    @classmethod
    def from_name(cls, name, *, create_if_missing=False, version=None, environment_name=None, **_kw):
        if name not in cls._named:
            cls._named[name] = cls(name)
        return cls._named[name]

    lookup = from_name

    @classmethod
    def ephemeral(cls, **_kw):
        import contextlib
        import tempfile

        @contextlib.contextmanager
        def cm():
            v = cls(f"ephemeral-{next(tempfile._get_candidate_names())}")
            try:
                yield v
            finally:
                shutil.rmtree(v.local_path, ignore_errors=True)

        return cm()

    def mount_at(self, path) -> bool:
        """Materialise ``volumes={path: vol}``: a virtual mount by default (see ``_mounts``), a symlink under
        ``MODAL_SHIM_MOUNTS=link``; returns whether ``path`` now resolves into the volume."""
        from . import _mounts

        return _mounts.register(path, self.local_path)

    def commit(self):
        return None

    def reload(self):
        return None

    def _abs(self, p):
        return os.path.join(self.local_path, str(p).lstrip("/"))

    def listdir(self, path="/", recursive=False):
        base = self._abs(path)
        out = []
        for root, dirs, files in os.walk(base):
            for n in dirs + files:
                out.append(_Entry(os.path.relpath(os.path.join(root, n), self.local_path)))
            if not recursive:
                break
        return out

    def read_file(self, path):
        with open(self._abs(path), "rb") as f:
            while chunk := f.read(1 << 20):
                yield chunk

    def remove_file(self, path, recursive=False):
        p = self._abs(path)
        shutil.rmtree(p) if os.path.isdir(p) else os.remove(p)

    def batch_upload(self, force=False):
        vol = self

        class _Up:
            def __enter__(s):
                return s

            def __exit__(s, *a):
                return False

            def put_file(s, local, remote):
                dst = vol._abs(remote)
                os.makedirs(os.path.dirname(dst), exist_ok=True)
                shutil.copy(local, dst) if isinstance(local, (str, os.PathLike)) else open(dst, "wb").write(local.read())

            def put_directory(s, local, remote, recursive=True):
                shutil.copytree(local, vol._abs(remote), dirs_exist_ok=True)

        return _Up()


@dataclass
class _Entry:
    path: str


class CloudBucketMount:
    def __init__(self, bucket_name=None, **kw):
        self.bucket_name, self.kw = bucket_name, kw


class NetworkFileSystem(Volume):
    pass


class Secret:
    def __init__(self, env=None, name=None):
        self._env, self.name = dict(env or {}), name

    @staticmethod
    def from_name(name, *, required_keys=None, environment_name=None, **_kw):
        return Secret({k: os.environ.get(k, "") for k in (required_keys or []) if k in os.environ}, name)

    @staticmethod
    def from_dict(d):
        return Secret({str(k): str(v) for k, v in dict(d or {}).items() if v is not None})

    @staticmethod
    def from_dotenv(*_a, **_k):
        return Secret({})

    @staticmethod
    def from_local_environ(keys):
        return Secret({k: os.environ[k] for k in keys if k in os.environ})


class Dict:
    _named: dict[str, "Dict"] = {}

    def __init__(self):
        self._d, self._lock = {}, threading.Lock()

    @classmethod
    def from_name(cls, name, *, create_if_missing=False, **_kw):
        if name not in cls._named:
            if not create_if_missing:
                raise NotFoundError(f"Dict {name!r} not found")
            cls._named[name] = cls()
        return cls._named[name]

    lookup = from_name

    @classmethod
    def ephemeral(cls, **_kw):
        import contextlib

        return contextlib.nullcontext(cls())

    def __getitem__(self, k):
        return self._d[k]

    def __setitem__(self, k, v):
        with self._lock:
            self._d[k] = v

    def __delitem__(self, k):
        with self._lock:
            del self._d[k]

    def __contains__(self, k):
        return k in self._d

    def get(self, k, default=None):
        return self._d.get(k, default)

    def put(self, k, v):
        self[k] = v

    def pop(self, k):
        with self._lock:
            return self._d.pop(k)

    def update(self, *a, **k):
        with self._lock:
            self._d.update(*a, **k)

    def keys(self):
        return list(self._d.keys())

    def values(self):
        return list(self._d.values())

    def items(self):
        return list(self._d.items())

    def len(self):
        return len(self._d)

    def clear(self):
        with self._lock:
            self._d.clear()


class Queue:
    _named: dict[str, "Queue"] = {}

    def __init__(self):
        self._parts = collections.defaultdict(_queue.Queue)

    @classmethod
    def from_name(cls, name, *, create_if_missing=False, **_kw):
        if name not in cls._named:
            if not create_if_missing:
                raise NotFoundError(f"Queue {name!r} not found")
            cls._named[name] = cls()
        return cls._named[name]

    lookup = from_name

    @classmethod
    def ephemeral(cls, **_kw):
        import contextlib

        return contextlib.nullcontext(cls())

    def put(self, v, *, partition=None, **_kw):
        self._parts[partition].put(v)

    def put_many(self, vs, *, partition=None, **_kw):
        for v in vs:
            self._parts[partition].put(v)

    def get(self, block=True, timeout=None, *, partition=None):
        try:
            return self._parts[partition].get(block=block, timeout=timeout)
        except _queue.Empty:
            return None

    def get_many(self, n_values, block=True, timeout=None, *, partition=None):
        out = []
        first = self.get(block, timeout, partition=partition)
        if first is None:
            return out
        out.append(first)
        while len(out) < n_values:
            try:
                out.append(self._parts[partition].get_nowait())
            except _queue.Empty:
                break
        return out

    def len(self, *, partition=None):
        return self._parts[partition].qsize()


@dataclass
class Retries:
    max_retries: int = 0
    backoff_coefficient: float = 2.0
    initial_delay: float = 1.0
    max_delay: float = 60.0


@dataclass
class Period:
    years: int = 0
    months: int = 0
    weeks: int = 0
    days: int = 0
    hours: int = 0
    minutes: int = 0
    seconds: float = 0


@dataclass
class Cron:
    cron_string: str = ""
    timezone: str = "UTC"


class Proxy:
    @staticmethod
    def from_name(name, **_kw):
        return Proxy()


class Sandbox:
    """OUT OF SCOPE (SURVEY.md §2.1 13_sandboxes): constructing one is an explicit error, not a silent no-op."""

    @staticmethod
    def create(*_a, **_k):
        raise NotImplementedError("modal.Sandbox is outside the in-box H100 runtime's scope")

    from_id = from_name = create
