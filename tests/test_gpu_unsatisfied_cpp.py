"""include/plonk_b200.hpp's debugger check (tests/cpp/unsatisfied_check.cpp): the reference's examples/circuit.rs with a
witness that breaks a range gate, as a Composer and against provers from compile and compile_with_compressed, name the same
failing range rows with one report; the honest witness reports nothing."""
import subprocess

import pytest

from tests.test_host_logic import _build_cpp


@pytest.mark.gpu
def test_cpp_mirror_reports_unsatisfied_constraints():
    out = subprocess.run([_build_cpp("unsatisfied_check")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert len(lines) == 13, lines
    bad, good = lines[:6], lines[6:12]
    # the three levels agree with each other, on the failing witness and on the honest one
    assert bad[0].split(" ", 1)[1] == bad[2].split(" ", 1)[1] == bad[4].split(" ", 1)[1]
    assert bad[1].split(" ", 1)[1] == bad[3].split(" ", 1)[1] == bad[5].split(" ", 1)[1]
    count = int(bad[0].split()[1])
    assert count >= 1
    first_row = bad[0].split()[2].split(":", 1)[0]
    report = bad[1].split(" ", 1)[1]
    assert report.startswith(f"plonk debugger: {count} of ") and report.endswith(" identity")
    assert f"; the first, constraint {first_row}, fails the " in report
    assert good == ["composer 0", "composer_report none", "prover 0", "prover_report none", "compressed 0", "compressed_report none"]
    assert lines[12] == "short_witness_table InvalidArgument"
