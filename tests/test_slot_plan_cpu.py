"""The slot planner of fyx_set_topology (fyrox_b200/csrc/fyx_slots.hpp): the (depth, parent slot, node index) order, level
offsets and parent slots, refused cycles, and the sub-forest groups and their selection rule, on random forests and
scenegen's scenes — tests/cpp/test_slot_plan.cpp, CPU only."""
import os
import subprocess


def test_slot_plan_layout_and_subforest_groups():
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp")
    subprocess.run(["make", "-C", d, "test_slot_plan"], check=True, capture_output=True)
    out = subprocess.run([os.path.join(d, "test_slot_plan")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "slot plan ok" in out.stdout
