"""`install_as_minimagen()` without the reference on the path; runs in a subprocess because it re-binds
sys.modules['minimagen*']."""
import os
import subprocess
import sys


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_install_as_minimagen_without_reference_is_alias_only():
    """No reference on the path: `minimagen` becomes an alias package of the hot-path modules only."""
    code = ("import sys; sys.path = [p for p in sys.path if 'reference' not in p]\n"
            "import minimagen_b200 as m; pkg = m.install_as_minimagen()\n"
            "from minimagen.Unet import Unet; from minimagen.Imagen import Imagen; from minimagen import Unet as U\n"
            "import minimagen_b200.Unet as MU\n"
            "assert Unet is MU.Unet and U is MU\n"
            "try:\n    import minimagen.generate\n    raise SystemExit('unexpected: minimagen.generate importable')\n"
            "except ModuleNotFoundError:\n    pass\nprint('ok')\n")
    env = dict(os.environ, PYTHONPATH=ROOT, MINIMAGEN_REFERENCE="/nonexistent")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=300, cwd="/tmp")
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stderr[-2000:]
