"""The signal and root-motion rules of fyrox_b200/csrc/fyx_anim_plan.hpp (event rings, draining, root-motion records and
refusals, group sources) — tests/cpp/test_anim_signal_plan.cpp, built with g++ into a temporary directory.  CPU only."""
import os
import subprocess
import tempfile


def test_anim_signal_plan_rules():
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "test_anim_signal_plan.cpp")
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "test_anim_signal_plan")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-Wall", "-o", exe, src], check=True, capture_output=True)
        out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "anim signal plan ok" in out.stdout
