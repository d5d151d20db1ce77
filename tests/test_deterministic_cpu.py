"""Deterministic mode without a GPU: the PFD_DETERMINISTIC switch, the Python API and the library options."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_env_flag_parsing():
    from pfd_b200 import native
    for v in ("1", "1 ", "10"):
        assert native.env_flag(v), v
    for v in (None, "", "0", "true", "yes", " 1"):
        assert not native.env_flag(v), v


def _mode_in_subprocess(env_value):
    env = {k: v for k, v in os.environ.items() if k != "PFD_DETERMINISTIC"}
    if env_value is not None:
        env["PFD_DETERMINISTIC"] = env_value
    code = "import pfd_b200; print(int(pfd_b200.is_deterministic()))"
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=ROOT, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout.strip().splitlines()[-1]


def test_environment_sets_the_default_mode():
    assert _mode_in_subprocess(None) == "0"
    assert _mode_in_subprocess("0") == "0"
    assert _mode_in_subprocess("1") == "1"


def test_set_deterministic_bumps_graph_generation():
    import pfd_b200
    from pfd_b200 import graphs
    was = pfd_b200.is_deterministic()
    try:
        g0 = graphs.generation()
        pfd_b200.set_deterministic(True)
        assert pfd_b200.is_deterministic() and graphs.generation() > g0
        g1 = graphs.generation()
        pfd_b200.set_deterministic(False)
        assert not pfd_b200.is_deterministic() and graphs.generation() > g1
    finally:
        pfd_b200.set_deterministic(was)


def test_raw_options_accepted_without_gpu():
    from pfd_b200 import native
    lib = native.load()
    try:
        for name, value in ((b"deterministic", 1), (b"deterministic", 0), (b"plan_sms", 114), (b"plan_sms", 0)):
            assert lib.pfd_set_option(name, value) == 0
        native.set_env_option("deterministic", 1)
        assert native.deterministic()
        native.set_env_option(None, None)                       # a reset returns to the environment's default
        assert native.deterministic() == native.env_flag(os.environ.get("PFD_DETERMINISTIC"))
    finally:
        native.set_env_option(None, None)
