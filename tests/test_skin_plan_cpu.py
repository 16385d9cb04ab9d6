"""The skinning-table planner of fyx_commit_surfaces (fyrox_b200/csrc/fyx_skin_plan.hpp): bone slots, k_skin's tiles, the
skinned-mesh fold with its late bones, and the bone-block tables, on random surface lists over random forests (with and
without a DFS rank) and on scenegen's skinned units — tests/cpp/test_skin_plan.cpp, CPU only."""
import os
import subprocess


def test_skin_plan_tables():
    d = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp")
    subprocess.run(["make", "-C", d, "test_skin_plan"], check=True, capture_output=True)
    out = subprocess.run([os.path.join(d, "test_skin_plan")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "skin plan ok" in out.stdout
