"""The problems per launch of the linear probe (gcc_b200.tasks.linear_probe.check_memory): all of them when the fit
fits in free device memory, fewer when only fewer fit (the result does not depend on it), the caller's choice when
given, and a refusal naming the sizes when even one problem per launch does not fit."""
import pytest

from gcc_b200 import _lib
from gcc_b200.tasks import linear_probe as lp


@pytest.fixture
def free_bytes(monkeypatch):
    box = {}
    monkeypatch.setattr(lp, "_free_bytes", lambda dev: box["free"])
    return box


def test_batch_follows_free_memory(free_bytes):
    n, d, c = 2_000_000, 256, 300                      # 3,000 problems at d = 256
    P = 10 * c
    full, one = lp.probe_bytes(n, d, c, 10, P), lp.probe_bytes(n, d, c, 10, 1)
    assert full > one
    free_bytes["free"] = full
    assert lp.check_memory(n, d, c) == P
    free_bytes["free"] = (full + one) // 2
    b = lp.check_memory(n, d, c)
    assert 1 <= b < P and lp.probe_bytes(n, d, c, 10, b) <= free_bytes["free"]
    assert lp.check_memory(n, d, c, batch=7) == 7
    free_bytes["free"] = one - 1
    with pytest.raises(_lib.GccbError, match=r"need [\d.]+ GB of device memory at 1 problem per launch"):
        lp.check_memory(n, d, c)
    with pytest.raises(_lib.GccbError, match="at 7 problems per launch"):
        lp.check_memory(n, d, c, batch=7)
