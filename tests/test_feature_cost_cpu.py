"""The binding's signature table and the A/B cost tool, without a GPU."""
import os
import subprocess
import sys

from conftest import ROOT
from raisimlib_b200 import capi


def test_every_exported_symbol_has_declared_argtypes():
    L = capi.lib()
    for name in capi.EXPORTED:
        assert getattr(L, name).argtypes is not None, name


def test_feature_cost_lists_every_feature_without_cuda():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "feature_cost.py"), "--list"], capture_output=True, text=True,
                         env=env, timeout=600)
    assert out.returncode == 0, out.stderr
    listed = {line.split()[0]: line for line in out.stdout.splitlines()}
    assert list(listed) == ["contact_forces", "body_inertia", "contact_friction", "actuator_params", "actuator_network", "actuation_delay",
                            "frame_kinematics", "height_scan", "terrain_curriculum"]
    assert listed["contact_forces"].endswith("modes none feet all all+read")
    assert listed["actuator_network"].endswith("modes pd limp net")
