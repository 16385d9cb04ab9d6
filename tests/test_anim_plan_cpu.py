"""N2's host rules (fyrox_b200/csrc/fyx_anim_plan.hpp): the per-node track order k_anim_apply blends in, on random animation
sets over random forests and on the bench's shape; every refusal of fyx_anim_add and fyx_anim_blend_group at its limit; the
track records; the time position against the oracle's wrapf — tests/cpp/test_anim_plan.cpp, CPU only."""
import os
import subprocess


def test_anim_plan_rules():
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp")
    subprocess.run(["make", "-C", d, "test_anim_plan"], check=True, capture_output=True)
    out = subprocess.run([os.path.join(d, "test_anim_plan")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "anim plan ok" in out.stdout
