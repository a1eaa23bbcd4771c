"""Sub-step barrier of a step launch that runs more than one round of warps (run on an H100: pytest -m gpu).

With more environments than resident warps, every warp runs one environment per round, and the warps of each round of a CTA
re-align at every sub-step, the barrier counting only the warps that own an environment in that round.  The alignment decides
when an environment is computed, never what: every result must be bit-identical to the same launches without the barrier.
"""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _outputs(sim, obs):
    bt = sim.bt
    g, v = bt.get_state()
    rec, cnt = bt.contacts()
    return dict(obs=obs.cpu().numpy(), gc=g, gv=v, contacts=rec, ncontacts=cnt, points=bt.contact_points(), iters=bt.solver_iterations(),
                resid=bt.solver_residual(), status=bt.solver_status(), tau=bt.generalized_force(), diverged=bt.diverged())


# 4096: the headline batch (a full second round on 124 of the 132 CTAs); 3001: a ragged second round (one CTA with 9 of its 16 warps)
@pytest.mark.parametrize("n", [4096, 3001])
def test_two_round_substep_barrier_is_bit_identical(monkeypatch, n):
    import torch
    import bench
    from raisimlib_b200 import capi
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    lib = capi.lib()
    lib.rsb_internal_launch_config.argtypes = [ctypes.c_void_p] * 3
    monkeypatch.setenv("RSB_FORCE_WPC", "16")
    stream = torch.cuda.current_stream()
    wl = bench.Workload("c3", 0, n)
    runs = []
    for barrier in ("1", "0"):
        monkeypatch.setenv("RSB_SUBSTEP_BARRIER", barrier)
        sim = bench.GpuSim(wl, 0, stream)
        wpc, grid = ctypes.c_int(), ctypes.c_int()
        assert lib.rsb_internal_launch_config(sim.bt.h, ctypes.byref(wpc), ctypes.byref(grid)) == 0
        assert wpc.value * grid.value < n < 2 * wpc.value * grid.value, "the batch must run in two rounds of warps"
        out = []
        for k in range(wl.settle + 6):       # robots land, then stand on the rough terrain under jittered targets
            obs = sim.step_resident(k)
            if k % 8 == 7 or k >= wl.settle:
                torch.cuda.synchronize()
                out.append(_outputs(sim, obs))
        runs.append(out)
        del sim
    assert runs[1][-1]["ncontacts"].mean() > 1.0, "the compared steps must exercise the contact solver"
    for k, (a, b) in enumerate(zip(*runs)):
        for name in a:
            assert a[name].shape == b[name].shape and a[name].tobytes() == b[name].tobytes(), \
                f"sample {k}: {name} differs between the launches with and without the sub-step barrier"
