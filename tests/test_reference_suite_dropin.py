"""The reference's OWN test-suite, unmodified and read in place, run against this package.

`tests/ref_suite_plugin.py` makes `import toppra` resolve to `toppra_b200`; pytest then collects the reference's test
files where they lie (`$TOPPRA_REFERENCE/tests/tests`, default /root/reference, or $TB_REFERENCE_TESTS) — nothing is
copied into this repository.
This is the drop-in claim in executable form: the reference's tests of its public API (interpolators, constraints,
solver-wrapper interface incl. `cy_seidel_solverwrapper.solve_lp1d / solve_lp2d / seidelWrapper`, TOPPRA / TOPPRAsd,
parametrizers, error behaviour) pass against toppra_b200.

Deselected, with the reason:
  * `qpoases`, `cvxpy`, and the `ecos` cases of test_basic_can_linear.py + test_ecos_wrapper.py — other solver BACKENDS of
    the reference (qpOASES / cvxpy / ECOS wrapper classes); this package has one backend ("seidel" == "b200"; a conic
    problem given "ecos" runs the robust scan, and that case, test_retime_wconic_constraints.py, IS run);
  * tests/cpp — the reference's C++ twin;
  * retime/robustness/test_robustness_main.py — selects the hotqpoases problems by default and writes a result file next to
    itself; its problem suite is covered by tests/golden/p4_robustness_suite.npz instead.
Tests that need OpenRAVE skip themselves, as they do for the reference.  Where the reference validates against cvxpy
(not installed here) tests/mini_cvxpy.py supplies the LP subset on scipy's HiGHS, so those tests validate against an
independent solver rather than skip.

Without a GPU the kernels are replaced by the oracle-backed double (tests/cpu_engine.py): what this run proves is the API
surface and the host logic.  The `gpu` variant runs the same suite on the real engine wherever a reference checkout is
available next to a GPU, and skips where there is none."""
import os
import re
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_TESTS = os.environ.get("TB_REFERENCE_TESTS", os.path.join(os.environ.get("TOPPRA_REFERENCE", "/root/reference"), "tests"))
SUITE = os.path.join(REF_TESTS, "tests")
DESELECT = "not qpoases and not cvxpy and not (test_basic_can_linear and ecos)"
IGNORE = ["cpp", "solverwrapper/test_ecos_wrapper.py", "retime/robustness/test_robustness_main.py"]
MIN_PASSED = 800     # 846 here; the exact count depends on which optional third-party packages are installed

needs_reference = pytest.mark.skipif(not os.path.isdir(SUITE), reason="no reference checkout at %s" % REF_TESTS)


def _run(engine):
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1", TB_REF_SUITE_ENGINE=engine,
               PYTHONPATH=os.pathsep.join([HERE, ROOT, os.environ.get("PYTHONPATH", "")]))
    cmd = [sys.executable, "-m", "pytest", "-p", "ref_suite_plugin", "-p", "no:cacheprovider", "--rootdir", REF_TESTS,
           "-q", "-W", "ignore", SUITE, "-k", DESELECT] + ["--ignore=" + os.path.join(SUITE, p) for p in IGNORE]
    proc = subprocess.run(cmd, env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    tail = "\n".join(proc.stdout.splitlines()[-40:])
    summary = proc.stdout.strip().splitlines()[-1]
    counts = {k: int(n) for n, k in re.findall(r"(\d+) (passed|failed|error|errors|skipped|deselected)", summary)}
    assert proc.returncode == 0, tail
    assert counts.get("failed", 0) == 0 and counts.get("error", 0) == 0 and counts.get("errors", 0) == 0, tail
    assert counts.get("passed", 0) >= MIN_PASSED, tail
    return counts


@needs_reference
def test_reference_suite_passes_against_toppra_b200_api():
    _run("cpu_double")


@pytest.mark.gpu
@needs_reference
def test_reference_suite_passes_on_the_gpu_engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    _run("gpu")


# ---- the reference's example scripts ----------------------------------------------------------------------------
EXAMPLES = os.environ.get("TB_REFERENCE_EXAMPLES", os.path.join(os.path.dirname(REF_TESTS.rstrip("/")), "examples"))
EXAMPLE_SCRIPTS = ["plot_scalar_example", "plot_straight_line", "plot_kinematics", "plot_kinematics_duration",
                   "plot_robust_kinematics"]
# compute_controllable_sets called AFTER other solves on the same instance: the reference's seidelWrapper carries its
# warm-start pair from call to call (pyx:526-527 zero it in __init__ only), this package starts every pass from zeros —
# a different but equally optimal start, so a few K entries move by one ulp.  First calls are bit-identical.
ULP_KEYS = {("plot_kinematics_duration", "K")}


def _run_examples(engine, tmp_path):
    """{script: npz dict} for `engine` and, where oracle/_ref is built, for the unmodified reference."""
    import numpy as np
    from oracle.ref_loader import reference_available
    runner = os.path.join(HERE, "ref_example_runner.py")
    engines = [engine] + (["reference"] if reference_available() else [])
    procs = {}
    for name in EXAMPLE_SCRIPTS:
        for eng in engines:
            if eng == "reference" and name == "plot_robust_kinematics":
                continue                      # needs ECOS, which is not installed: nothing to compare with
            out = str(tmp_path / ("%s_%s.npz" % (name, eng)))
            procs[name, eng] = (out, subprocess.Popen(
                [sys.executable, runner, eng, os.path.join(EXAMPLES, name + ".py"), out], cwd=ROOT,
                env=dict(os.environ, PYTHONDONTWRITEBYTECODE="1"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    results = {}
    for (name, eng), (out, proc) in procs.items():
        log = proc.communicate(timeout=900)[0]
        assert proc.returncode == 0, "%s on %s:\n%s" % (name, eng, "\n".join(log.splitlines()[-25:]))
        results[name, eng] = dict(np.load(out))
    return results, engines


def _check_examples(engine, tmp_path):
    import numpy as np
    results, engines = _run_examples(engine, tmp_path)
    for name in EXAMPLE_SCRIPTS:
        mine = results[name, engine]
        assert np.isfinite(mine["jnt_traj__duration"]) and mine["jnt_traj__duration"] > 0, name
        if (name, "reference") not in results:
            continue
        ref = results[name, "reference"]
        assert set(mine) == set(ref), (name, sorted(set(mine) ^ set(ref)))
        for key in ref:
            if (name, key) in ULP_KEYS:
                np.testing.assert_allclose(mine[key], ref[key], rtol=1e-13, atol=0, err_msg="%s %s" % (name, key))
            else:
                assert np.array_equal(mine[key], ref[key]), (name, key)
    robust = results["plot_robust_kinematics", engine]             # BASELINE cfg 4's script: solved, sets well-formed
    assert robust["sd_vec"].shape == (101,) and np.all(robust["K"][:, 0] <= robust["K"][:, 1] + 1e-12)
    assert np.all(robust["X"][:, 1] + 1e-9 >= robust["K"][:, 1])


@pytest.mark.skipif(not os.path.isdir(EXAMPLES), reason="no reference examples at %s" % EXAMPLES)
def test_reference_examples_run_unmodified_and_match_the_reference(tmp_path):
    """examples/*.py of the reference (BASELINE cfg 1 = plot_kinematics.py, cfg 4 = plot_robust_kinematics.py), run as
    they are with `toppra` -> toppra_b200: every number they compute is IDENTICAL to what the unmodified reference build
    computes from the same script (one documented one-ulp exception, ULP_KEYS)."""
    _check_examples("cpu_double", tmp_path)


@pytest.mark.gpu
@pytest.mark.skipif(not os.path.isdir(EXAMPLES), reason="no reference examples at %s" % EXAMPLES)
def test_reference_examples_on_the_gpu_engine(tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    _check_examples("gpu", tmp_path)
