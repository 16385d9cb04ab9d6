"""Dynamic batching's host rules (fyrox_b200/csrc/fyx_dyn_plan.hpp): the device tables in push order on random registrations
and quad nodes over random forests; every refusal of fyx_add_dynamic_surface and fyx_set_sprites at its limit; the release of
ids and keys; the pools' compaction; the placement of a pack's segments at its size limits — tests/cpp/test_dyn_plan.cpp,
CPU only."""
import os
import subprocess


def test_dyn_plan_rules():
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp")
    subprocess.run(["make", "-C", d, "test_dyn_plan"], check=True, capture_output=True)
    out = subprocess.run([os.path.join(d, "test_dyn_plan")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "dyn plan ok" in out.stdout
