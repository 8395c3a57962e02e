"""engine.run_each, the fan-out over the engines that the reference load, the batch loop and the BGZF and BAM writers use."""
import threading
import time

import pytest


def test_run_each():
    """n == 0 calls nothing, n == 1 calls work(0) on the caller's thread, more run side by side, one thread each.  Every
    call ends before the exception of the lowest k that raised one (not the first raised) is re-raised on the caller's
    thread."""
    from badread_b200.engine import run_each
    run_each(0, lambda k: pytest.fail('called with n == 0'))
    me, seen = threading.current_thread(), []
    run_each(1, lambda k: seen.append((k, threading.current_thread() is me)))
    assert seen == [(0, True)]

    together, done = threading.Barrier(4, timeout=30), []

    def work(k):
        assert threading.current_thread() is not me
        together.wait()   # (all four at once)
        time.sleep({0: 0.2, 1: 0.1}.get(k, 0))
        if k in (1, 3):
            raise ValueError(k)
        done.append(k)

    with pytest.raises(ValueError) as e:
        run_each(4, work)
    assert e.value.args == (1,)
    assert sorted(done) == [0, 2]
