"""The packing core both engines share (medaka_b200/csrc/packing.h), driven on the CPU by a fake engine
(tests/native/packing_check.cpp) that logs the core's open, stage and launch calls."""
import os
import shutil
import subprocess

import pytest

from tests.test_read_level_engine import CALLS, P0, P1, TAIL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# test_forward_dev.py::test_forward_dev_packed_matches_host_forwards: (windows, columns) of its device calls
FORWARD_DEV_PLAN = [(150, 2000), (30, 2000), (40, 2000), (1, 2000), (400, 2000), (500, 2000), (20, 2000),
                    (200, 1500), (25, 1500), (60, 1500), (5, 1500)]


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    cxx = os.environ.get("CXX") or shutil.which("c++") or shutil.which("g++")
    exe = str(tmp_path_factory.mktemp("packing") / "packing_check")
    subprocess.run([cxx, "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe,
                    os.path.join(ROOT, "tests", "native", "packing_check.cpp")], check=True)

    def run(*commands):
        r = subprocess.run([exe], input="\n".join(commands) + "\n", capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        return r.stdout.splitlines()
    return run


def _launches(log):
    """(serial, length, [(call, first, n), ...]) of every launched group, in launch order."""
    out = []
    for line in log:
        if line.startswith("launch "):
            f = line.split()
            pieces = [tuple(int(v) for v in p.replace(":", " ").replace("+", " ").split()) for p in f[4:]]
            assert sum(n for _, _, n in pieces) == int(f[3]), line
            out.append((int(f[1]), int(f[2]), pieces))
    return out


def _expected(calls, gmax):
    """Groups by the protocol's rules: windows of consecutive calls fill groups of gmax; a new length seals the open
    group; a call of more than gmax windows runs as a group of its own.  Returns (launched groups, the open group)."""
    done, cur, length = [], [], None

    def seal():
        if cur:
            done.append((len(done), length, list(cur)))
            cur.clear()
    for i, (B, L) in enumerate(calls):
        if L != length:
            seal()
            length = L
        if B > gmax:
            seal()
            done.append((len(done), L, [(i, 0, B)]))
            continue
        first = 0
        while first < B:
            n = min(gmax - sum(p[2] for p in cur), B - first)
            cur.append((i, first, n))
            first += n
            if sum(p[2] for p in cur) == gmax:
                seal()
    return done, cur


def _commands(calls, gmax):
    return ["gmax %d" % gmax] + ["%s %d %d" % ("alone" if B > gmax else "call", B, L) for B, L in calls]


def _check_stages(log):
    """Each piece is staged at the group's window count so far."""
    at = 0
    for line in log:
        f = line.split()
        if f[0] == "open":
            at = 0
        elif f[0] == "stage":
            assert int(f[4]) == at, line
            at += int(f[3])


@pytest.mark.parametrize("gmax", [112, 64])
def test_read_level_engine_calls(driver, gmax):
    calls = [(B, P0) for B, _ in CALLS] + [(B, P1) for B, _ in TAIL]
    log = driver(*_commands(calls, gmax))
    want, still_open = _expected(calls, gmax)
    assert _launches(log) == want
    assert sum(n for _, _, n in want[0][2]) == gmax
    assert want[0][2][-1][1] == 0 and want[1][2][0][1] > 0           # a call straddles the first two groups
    assert len(want) == (2 if gmax == 112 else 3)
    assert still_open == [(len(CALLS), 0, TAIL[0][0]), (len(CALLS) + 1, 0, TAIL[1][0])]   # the tail stays open
    _check_stages(log)
    log = driver(*(_commands(calls, gmax) + ["flush"]))
    assert _launches(log)[-1] == (len(want), P1, still_open)


@pytest.mark.parametrize("gmax", [48, 1056])
def test_forward_dev_plan(driver, gmax):
    log = driver(*(_commands(FORWARD_DEV_PLAN, gmax) + ["flush"]))
    want, still_open = _expected(FORWARD_DEV_PLAN, gmax)
    assert _launches(log) == want + [(len(want), FORWARD_DEV_PLAN[-1][1], still_open)]
    _check_stages(log)
    if gmax == 1056:   # the 500-window call is split by the first full group, the column change seals the second
        assert want[0][2][-1] == (5, 0, 435) and want[1][2] == [(5, 435, 65), (6, 0, 20)] and len(want) == 2


def test_length_change_seals_the_group(driver):
    log = driver("gmax 100", "call 3 10", "call 2 20")
    assert log == ["open 3", "stage 0 0 3 0", "ticket 0", "launch 0 10 3 0:0+3", "open 2", "stage 1 0 2 0", "ticket 1"]


def test_oversized_call_forms_one_group(driver):
    log = driver("gmax 48", "call 10 7", "alone 500 7", "call 5 7")
    assert _launches(log) == [(0, 7, [(0, 0, 10)]), (1, 7, [(1, 0, 500)])]
    assert "open 500" in log


def test_fresh_group_takes_one_window(driver):
    log = driver("gmax 8", "cap 0", "call 3 5")
    assert _launches(log) == [(0, 5, [(0, 0, 1)]), (1, 5, [(0, 1, 1)]), (2, 5, [(0, 2, 1)])]
    assert [line for line in log if line.startswith("open")] == ["open 3", "open 2", "open 1"]


def test_wait_on_an_open_group_launches_it(driver):
    log = driver("gmax 16", "call 10 5", "call 10 5", "wait 1", "wait 0", "wait 1")
    assert log[-4:] == ["launch 1 5 4 1:6+4", "wait 1 1", "wait 0 0", "wait 1 1"]    # launched once
    assert _launches(log) == [(0, 5, [(0, 0, 10), (1, 0, 6)]), (1, 5, [(1, 6, 4)])]


def test_wait_on_a_ticket_older_than_the_ring(driver):
    """5000 one-window calls into one 10 000-window group: ticket 0 has left the 4096-entry ring, yet its group is still
    open.  The wait launches it and names it, rather than returning as if it had completed."""
    log = driver(*(["gmax 10000"] + ["call 1 3"] * 5000 + ["wait 0"]))
    assert log[-2].startswith("launch 0 3 5000 0:0+1 1:0+1 ")
    assert log[-1] == "wait 0 0"
