"""``gpu=`` grammar (SURVEY.md §2.2): "H100", "a10g", "A100-80GB", "H100:2", f"B200:{N}", "H100!", "any",
lists of fallbacks, ``modal.gpu.L40S(count=N)``, None/False.  In-box every value means "N of the local H100s"."""
from __future__ import annotations


class _GPU:
    def __init__(self, count: int = 1, **_kw):
        self.count = int(count)

    def __repr__(self):
        return f"modal.gpu.{type(self).__name__}(count={self.count})"


for _n in ("T4", "L4", "A10G", "A100", "H100", "H200", "B200", "L40S", "Any"):
    globals()[_n] = type(_n, (_GPU,), {})


def parse_gpu_count(spec) -> int:
    """Number of GPUs a ``gpu=`` value asks for (0 for None/False)."""
    if spec is None or spec is False:
        return 0
    if isinstance(spec, (list, tuple)):
        return parse_gpu_count(spec[0]) if spec else 0
    if isinstance(spec, _GPU):
        return spec.count
    s = str(spec).strip().rstrip("!")
    if ":" in s:
        name, _, cnt = s.partition(":")
        try:
            return max(1, int(cnt))
        except ValueError:
            raise ValueError(f"bad gpu spec {spec!r}") from None
    return 1
