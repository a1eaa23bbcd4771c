"""The C++ facade's traffic with the C ABI, on the CPU: tests/cpp/facade_trace.cpp drives the raisim:: headers against a recording stub of
include/rsb.h (tests/cpp/rsb_recording_stub.cpp), built with g++ alone (no CUDA, no librsb), and the log of rsb_batch_* calls is checked.

The goldens tests/golden/facade_trace_{standalone,vecenv}.txt were generated from the headers of the commit before the facade's accessors
got one code path (the stand-alone and lock-step branches of every accessor), so they record what each accessor issued then:

    git worktree add /tmp/parent <that commit> && g++ -std=c++17 -Wall -O1 -I/tmp/parent/include -o facade_trace \\
        tests/cpp/facade_trace.cpp tests/cpp/rsb_recording_stub.cpp && ./facade_trace standalone > tests/golden/facade_trace_standalone.txt
    (and the same with `vecenv`)

The vecenv scenario avoids the four getters that read the device without bringing the lock-step mirror up to date before (getMassMatrix,
getNonlinearities, getPosition, getLoopCounter); the sync scenario checks that they now do."""
import os
import subprocess

import pytest

from conftest import ROOT

CPP = os.path.join(ROOT, "tests", "cpp")
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def trace(tmp_path_factory):
    exe = tmp_path_factory.mktemp("facade_trace") / "facade_trace"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-o", str(exe),
                           os.path.join(CPP, "facade_trace.cpp"), os.path.join(CPP, "rsb_recording_stub.cpp")])

    def run(scenario):
        out = subprocess.run([str(exe), scenario], capture_output=True, text=True, timeout=60)
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr
        return out.stdout
    return run


@pytest.mark.parametrize("scenario", ["standalone", "vecenv"])
def test_facade_trace_matches_golden(trace, scenario):
    """every C-ABI call of a stand-alone World and of a 3-environment VectorizedEnvironment (arguments, buffer contents, order), and every
    value their getters return, equal the recorded log"""
    with open(os.path.join(GOLDEN, f"facade_trace_{scenario}.txt")) as f:
        want = f.read()
    got = trace(scenario)
    assert got.splitlines() == want.splitlines()


def test_standalone_control_step_calls(trace):
    """a stand-alone control step (setPdTarget, 4 x integrate(), getState) is one target upload, four launches (each followed by the
    world-time read of the time step) and one state read"""
    log = trace("standalone").splitlines()
    steps = 0
    for i, line in enumerate(log):
        if line != "# control step":
            continue
        calls = [l.split()[0] for l in log[i + 1: log.index("# end control step", i)]]
        assert calls == ["rsb_batch_set_pd_target"] + ["rsb_batch_integrate", "rsb_batch_get_params"] * 4 + ["rsb_batch_get_state"]
        steps += 1
    assert steps == 3


def _phases(log):
    """the log split at its '# ...' lines: [(phase, [call names])]"""
    out = []
    for line in log.splitlines():
        if line.startswith("# "):
            out.append((line[2:], []))
        elif line.startswith("rsb_"):
            out[-1][1].append(line.split()[0])
    return out


def test_lockstep_device_getters_see_pending_work(trace):
    """inside a VectorizedEnvironment, getMassMatrix / getNonlinearities / getPosition / getLoopCounter after integrate() read the state
    of the fused launch: the uploads and the launch come first in the log.  In reset(), getMassMatrix after setState reads the new state:
    the state upload comes first"""
    phases = _phases(trace("sync"))
    step_getters = ["rsb_batch_get_mass_matrix", "rsb_batch_get_nonlinearities", "rsb_batch_get_body_poses", "rsb_batch_get_solver_iterations"]
    checked = 0
    for i, (name, calls) in enumerate(phases):
        if name == "step 1":       # the last environment's fiber: the launch happens when it asks, then both environments read
            assert calls[:3] == ["rsb_batch_set_pd_target", "rsb_batch_set_generalized_force", "rsb_batch_integrate"]
            assert calls[3:] == step_getters + ["rsb_batch_get_state"] + step_getters
            assert all(c == "rsb_batch_get_params" for c in phases[i - 1][1])   # environment 0 read nothing before the launch
            checked += 1
        if name.startswith("reset "):
            assert calls[-2:] == ["rsb_batch_set_state", "rsb_batch_get_mass_matrix"]
            checked += 1
    assert checked == 3 + 2 * 2      # three steps, init and the final reset of two environments


def test_examples_compile_against_the_facade(tmp_path):
    """every example that uses the facade compiles against the headers (syntax only: no librsb needed)"""
    ex = os.path.join(ROOT, "examples")
    for name in sorted(os.listdir(ex)):
        if name.endswith(".cpp") and name != "multi_gpu.cpp":      # multi_gpu uses the C ABI and the CUDA runtime only
            subprocess.check_call(["g++", "-fsyntax-only", "-std=c++17", "-Wall", "-Werror", "-I" + os.path.join(ROOT, "include"), "-I" + ex,
                                   os.path.join(ex, name)])
