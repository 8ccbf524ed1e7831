"""Which loads time the launch plans instead of taking the built-in planner's choice (measure_plan_at_load), on the CPU."""
import subprocess


def test_only_large_unpinned_single_device_handles_time_their_plans():
    """tools/plan_check trigger prints the decision for every DTE_TUNE pin, forced variant, handle kind and workload hint.
    A handle times its plans only when nothing pins the plan (chunk only sizes the landing slots), no kernel variant is
    forced, it drives one device and it was configured for at least 8 M tuples; every other handle keeps the static plan
    that tests/golden/plan_table.txt.xz describes."""
    from ddt_b200 import build as B
    out = subprocess.run([B.build_plan_check(), "trigger"], capture_output=True, text=True, timeout=60)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.splitlines()
    assert len(lines) == 9 * 4 * 2 * 5
    measured = 0
    for line in lines:
        tune, want, multi, hint, got = line.split(" ")
        expect = tune in ("DTE_TUNE=", "DTE_TUNE=chunk=65536") and want == "0" and multi == "0" and int(hint) >= 8_000_000
        assert got == ("1" if expect else "0"), line
        measured += expect
    assert measured == 4
