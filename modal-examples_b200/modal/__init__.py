"""In-box ``modal``: the Python surface the reference scripts are written against (``modal-labs/modal-examples``,
census in SURVEY.md §2.2), executing on the local multi-H100 host instead of the Modal cloud.  GPU work goes through
``b200rt`` (ctypes over ``libb200rt.so``); everything that only makes sense in the cloud (images, secrets stores,
web endpoints, schedules) is accepted and inert so that scripts import and run unchanged."""
from . import config, exception, experimental, gpu  # noqa: F401
from ._runtime import is_local
from .app import App, Stub, enable_output
from .cls import Cls, batched, concurrent, enter, exit, method, parameter  # noqa: A004
from .functions import Function, FunctionCall
from .image import Image
from .resources import (CloudBucketMount, Cron, Dict, NetworkFileSystem, Period, Proxy, Queue, Retries, Sandbox, Secret,
                        Volume)
from .web import asgi_app, fastapi_endpoint, web_endpoint, web_server, wsgi_app

__version__ = "0.0.0+b200.inbox"

__all__ = [
    "App", "Stub", "Cls", "Function", "FunctionCall", "Image", "Volume", "Secret", "Dict", "Queue", "CloudBucketMount",
    "NetworkFileSystem", "Period", "Cron", "Retries", "Proxy", "Sandbox", "method", "enter", "exit", "parameter", "concurrent",
    "batched", "asgi_app", "wsgi_app", "fastapi_endpoint", "web_endpoint", "web_server", "is_local", "enable_output", "config",
    "exception", "experimental", "gpu",
]
