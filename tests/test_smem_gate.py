"""CPU: the cudaFuncSetAttribute interposer that test_gpu_threads.py preloads (tests/gate/smem_gate.c) holds, releases
and times out as that test relies on, so a broken gate shows without a device.

Each case runs in a fresh interpreter that loads the gate alone: its counters start at zero, and no CUDA runtime stands
behind it, so every set returns cudaErrorUnknown (999) after the gate has done its part.  One case loads the library
under test as well, to see that the gate then finds the runtime it brings in.  The kernels are two distinct
addresses; nothing dereferences them."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE = os.path.join(ROOT, "tests", "gate", "libsmem_gate.so")
ATTR = 8   # cudaFuncAttributeMaxDynamicSharedMemorySize

PRELUDE = f"""
import ctypes as C, json, threading, time
g = C.CDLL({GATE!r})
g.cudaFuncSetAttribute.argtypes = [C.c_void_p, C.c_int, C.c_int]
K1, K2 = C.c_void_p(0x1000), C.c_void_p(0x2000)
def stats():
    n = [C.c_int() for _ in range(3)]
    g.gate_stats(*(C.byref(x) for x in n))
    return dict(zip(("holds", "releases", "timeouts"), (x.value for x in n)))
def timed_set(k, value, attr={ATTR}, out=None):
    t = time.monotonic()
    rc = g.cudaFuncSetAttribute(k, attr, value)
    ms = (time.monotonic() - t) * 1e3
    if out is not None:
        out.update(rc=rc, ms=ms)
    return rc, ms
"""


def run(body):
    """body after PRELUDE in a fresh interpreter; it prints one JSON line -> that object"""
    code = PRELUDE + textwrap.dedent(body)
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=60)
    assert p.returncode == 0, p.stderr
    return json.loads(p.stdout.strip().splitlines()[-1])


@pytest.fixture(scope="module", autouse=True)
def gate_built():
    assert os.path.exists(GATE), f"{GATE} is missing: __graft_entry__.build() makes it (make -C tests/gate)"


def test_forwards_to_a_runtime_loaded_with_dlopen():
    """the library under test links the runtime and comes in through ctypes.CDLL, outside the global scope: the gate must
    still find the runtime's cudaFuncSetAttribute, or every set would fail with cudaErrorUnknown"""
    lib = os.path.join(ROOT, "primestereomatch_b200", "libprime_stereo_b200.so")
    r = run(f"""
        before = g.gate_forwards()
        C.CDLL({lib!r})
        print(json.dumps(dict(before=before, after=g.gate_forwards())))
    """)
    assert r == {"before": 0, "after": 1}, r


def test_unarmed_and_small_sets_pass_through():
    r = run("""
        a = timed_set(K1, 65536)                 # not armed
        g.gate_arm(60000, 2000)
        b = timed_set(K1, 49152)                 # below the armed size
        c = timed_set(K1, 65536, attr=9)         # another attribute (the preferred carveout)
        print(json.dumps(dict(a=a, b=b, c=c, still_armed=not g.gate_wait_held(50), **stats())))
    """)
    for k in "abc":
        assert r[k][0] == 999, r                  # forwarded: no runtime behind the gate here
        assert r[k][1] < 500, r
    assert r["still_armed"], "a set the gate must ignore disarmed it"
    assert (r["holds"], r["releases"], r["timeouts"]) == (0, 0, 0), r


def test_hold_ends_at_its_timeout():
    r = run("""
        g.gate_arm(60000, 300)
        rc, ms = timed_set(K1, 65536)
        again = timed_set(K1, 65536)             # one hold per arming
        print(json.dumps(dict(rc=rc, ms=ms, again=again, **stats())))
    """)
    assert r["rc"] == 999
    assert 250 <= r["ms"] < 5000, r
    assert r["again"][1] < 250, "the gate held twice for one arming"
    assert (r["holds"], r["releases"], r["timeouts"]) == (1, 0, 1), r


def test_hold_ends_when_another_thread_sets_the_same_kernel():
    r = run("""
        g.gate_arm(60000, 10000)
        held = {}
        t = threading.Thread(target=timed_set, args=(K1, 65536), kwargs={"out": held})
        t.start()
        began = g.gate_wait_held(5000)
        other = timed_set(K2, 49152)             # another kernel: the hold goes on
        time.sleep(0.2)
        alive_after_other = t.is_alive()
        mine = timed_set(K1, 49152)              # the same kernel from this thread: released
        t.join(10)
        print(json.dumps(dict(began=began, alive_after_other=alive_after_other, other=other, mine=mine,
                              held=held, **stats())))
    """)
    assert r["began"] == 1, r
    assert r["alive_after_other"], "a set of another kernel ended the hold"
    assert r["other"][1] < 500 and r["mine"][1] < 500, "only the armed set may wait"
    assert r["held"]["rc"] == 999 and 200 <= r["held"]["ms"] < 5000, r
    assert (r["holds"], r["releases"], r["timeouts"]) == (1, 1, 0), r


def test_wait_held_times_out_when_nothing_reaches_the_gate():
    r = run("""
        g.gate_arm(60000, 1000)
        t = time.monotonic()
        began = g.gate_wait_held(100)
        print(json.dumps(dict(began=began, ms=(time.monotonic() - t) * 1e3, **stats())))
    """)
    assert r["began"] == 0 and 90 <= r["ms"] < 5000, r
    assert r["holds"] == 0, r
