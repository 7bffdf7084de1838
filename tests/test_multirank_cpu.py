"""tests/multirank.py's runner with small python processes: every rank's environment and output; a failed rank, or the
timeout, ends the run at once with every rank killed and reaped."""
import subprocess
import sys
import time

import pytest

import multirank as mr


def _python(code):
    return [sys.executable, "-c", code]


@pytest.fixture
def started(monkeypatch):
    """the processes the runner starts"""
    procs = []

    class Recorded(subprocess.Popen):
        def __init__(self, *args, **kw):
            super().__init__(*args, **kw)
            procs.append(self)
    monkeypatch.setattr(subprocess, "Popen", Recorded)
    return procs


def test_every_rank_exits_zero(started):
    logs = mr.run(2, lambda r: _python("import os; print(%d, os.environ['RANK'], os.environ['WORLD_SIZE'])" % r))
    assert [log.split() for log in logs] == [["0", "0", "2"], ["1", "1", "2"]]
    assert [p.returncode for p in started] == [0, 0]


def test_a_failed_rank_ends_the_run(started):
    t0 = time.monotonic()
    with pytest.raises(AssertionError, match=r"a rank failed; exit codes \[-9, 1\]") as e:
        mr.run(2, lambda r: _python("import time; time.sleep(60)" if r == 0 else "print('rank 1 fails'); exit(1)"))
    assert time.monotonic() - t0 < 10
    assert "rank 1 fails" in str(e.value)
    assert len(started) == 2 and all(p.poll() is not None for p in started)


def test_the_timeout_ends_the_run(started):
    t0 = time.monotonic()
    with pytest.raises(AssertionError, match=r"timed out after 1 s; exit codes \[-9, -9\]"):
        mr.run(2, lambda r: _python("import time; time.sleep(60)"), timeout=1)
    assert time.monotonic() - t0 < 10
    assert len(started) == 2 and all(p.poll() is not None for p in started)
