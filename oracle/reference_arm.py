"""Install the UNMODIFIED reference package into the git-ignored oracle/_ref, for the reference arm of bench.py
(`--impl reference`, `cpu_baseline.kind = "reference"`) and tools/compare_reference_gpu.py.

build() runs it.  The reference sources are its `inference_lib` directory: $AQLM_REFERENCE_SRC when set, otherwise the first
of the reference checkout's usual locations that exists (beside this repository, or /root/reference).  Without them
nothing is installed and bench.py times the oracle's C port instead.  Never fatal."""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "_ref")
DEFAULT_SOURCES = (os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference", "inference_lib"),
                   "/root/reference/inference_lib")


def source_dir():
    """The reference's inference_lib directory, or None."""
    env = os.environ.get("AQLM_REFERENCE_SRC")
    for d in ((env,) if env else DEFAULT_SOURCES):
        if os.path.isfile(os.path.join(d, "setup.cfg")) or os.path.isfile(os.path.join(d, "pyproject.toml")):
            return d
    return None


def install() -> None:
    src = source_dir()
    if os.path.isdir(os.path.join(TARGET, "aqlm")) or src is None:
        return
    tmp = tempfile.mkdtemp(prefix="aqlm_ref_src_")
    try:  # the reference tree may be read-only and setuptools writes egg-info into the source tree: install from a copy
        shutil.copytree(src, os.path.join(tmp, "inference_lib"))
        subprocess.check_call([sys.executable, "-m", "pip", "install", "-q", "--no-index", "--no-build-isolation", "--no-deps",
                               "--target", TARGET, os.path.join(tmp, "inference_lib")])
        print("reference arm installed:", TARGET)
    except Exception as e:
        print("note: reference arm not installed:", e)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
