"""Build recipe of the reference binaries the tests compare against (written to oracle/_ref/, git-ignored).

    python -m oracle.build_ref

mise: the reference's MISE octree (code/lib/libmise/mise.pyx) is cythonized and compiled with g++ against the Python
headers into oracle/_ref/mise*.so.  The reference tree is read in place; nothing from it is copied into the
repository.  When the tree is absent the recipe skips, and the module built earlier (if any) is used as it is.
"""
import os
import shutil
import subprocess
import sys
import sysconfig

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_ref")
REFERENCE = os.environ.get("MP_REFERENCE", "/root/reference")
MISE_PYX = os.path.join(REFERENCE, "code", "lib", "libmise", "mise.pyx")


def mise_path():
    """Path of the built module, or None."""
    p = os.path.join(OUT, "mise" + sysconfig.get_config_var("EXT_SUFFIX"))
    return p if os.path.exists(p) else None


def build_mise(force=False):
    so = os.path.join(OUT, "mise" + sysconfig.get_config_var("EXT_SUFFIX"))
    if not os.path.exists(MISE_PYX):
        return mise_path()
    if os.path.exists(so) and not force and os.path.getmtime(so) >= os.path.getmtime(MISE_PYX):
        return so
    import numpy as np
    os.makedirs(OUT, exist_ok=True)
    tmp = os.path.join(OUT, "mise_build")
    os.makedirs(tmp, exist_ok=True)
    pyx = os.path.join(tmp, "mise.pyx")
    shutil.copyfile(MISE_PYX, pyx)
    cpp = os.path.join(tmp, "mise.cpp")
    subprocess.check_call([sys.executable, "-m", "cython", "-3", "--cplus", pyx, "-o", cpp],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    cxx = os.environ.get("CXX", "g++")
    subprocess.check_call([cxx, "-O2", "-shared", "-fPIC", "-w", "-I", sysconfig.get_paths()["include"],
                           "-I", np.get_include(), cpp, "-o", so])
    shutil.rmtree(tmp, ignore_errors=True)
    return so


def load_mise():
    """The compiled reference module (``mise.MISE``), or None when it has not been built."""
    p = mise_path()
    if p is None:
        return None
    import importlib.util
    spec = importlib.util.spec_from_file_location("mise", p)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def build(force=False):
    return build_mise(force)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
