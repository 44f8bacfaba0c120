"""Builds oracle/_ref/esac_ref*.so: the reference's OWN esac extension, compiled from its unmodified sources where a
checkout of vislearn/esac is named by $ESAC_REFERENCE or sits beside the repository as `reference` (code/esac: esac.cpp,
thread_rand.cpp + the four headers they include), against the minimal OpenCV stand-in of oracle/ref_shim/ (whose calib3d
calls are executed by the real OpenCV inside the cv2 wheel).

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Nothing from the reference is copied into the repository; outputs go to
oracle/_ref/ only (git-ignored).  The reference's own build system (code/esac/setup.py) is not run: it needs $CONDA_PREFIX
and the OpenCV C++ headers / libraries.

    [ESAC_REFERENCE=<checkout of vislearn/esac>] python -m oracle.build_ref [--force]
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
SHIM = HERE / "ref_shim"
OUT_DIR = HERE / "_ref"


def _find_reference() -> Path | None:
    """code/esac of the reference checkout: the one $ESAC_REFERENCE names, else a checkout named `reference` beside this
    repository or beside one of its enclosing directories (the nearest wins)."""
    if os.environ.get("ESAC_REFERENCE"):
        return Path(os.environ["ESAC_REFERENCE"]) / "code" / "esac"
    for d in HERE.parent.parents:
        cand = d / "reference" / "code" / "esac"
        if cand.is_dir():
            return cand
    return None


REF_SRC = _find_reference()
REF_FILES = ["esac.cpp", "thread_rand.cpp", "thread_rand.h", "esac_types.h", "esac_util.h", "esac_loss.h",
             "esac_derivative.h", "stop_watch.h"]
SHIM_FILES = [SHIM / "opencv2" / "opencv.hpp", SHIM / "shim_cv2.cpp", SHIM / "ref_module.cpp"]
CXX = "/usr/bin/g++"


def lib_path() -> Path:
    return OUT_DIR / ("esac_ref" + sysconfig.get_config_var("EXT_SUFFIX"))


def reference_available() -> bool:
    return REF_SRC is not None and all(os.access(REF_SRC / f, os.R_OK) for f in REF_FILES)


def _digest() -> str:
    h = hashlib.sha256()
    for p in SHIM_FILES + [REF_SRC / f for f in REF_FILES]:
        h.update(p.name.encode())
        h.update(p.read_bytes())
    return h.hexdigest()


def build_ref(force: bool = False, verbose: bool = False) -> Path | None:
    """Returns the path of the built module, or None when the reference sources are absent (or unreadable) and nothing
    was built before."""
    lib = lib_path()
    if not reference_available():
        return lib if lib.exists() else None
    OUT_DIR.mkdir(exist_ok=True)
    stamp = OUT_DIR / "esac_ref.srchash"
    want = _digest()
    if not force and lib.exists() and stamp.exists() and stamp.read_text().strip() == want:
        return lib
    import torch
    from torch.utils import cpp_extension as ce
    inc = [f"-I{SHIM}", f"-I{REF_SRC}"] + [f"-isystem{p}" for p in ce.include_paths()] + [f"-isystem{sysconfig.get_paths()['include']}"]
    common = ["-std=c++17", "-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-w",
              f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}", "-DTORCH_API_INCLUDE_EXTENSION_H"]
    jobs = [
        # the reference's own pybind module in esac.cpp gets a throw-away name; ref_module.cpp binds the same functions
        (REF_SRC / "esac.cpp", ["-DTORCH_EXTENSION_NAME=esac_ref_unused"]),
        (REF_SRC / "thread_rand.cpp", []),
        (SHIM / "shim_cv2.cpp", []),
        (SHIM / "ref_module.cpp", ["-DTORCH_EXTENSION_NAME=esac_ref"]),
    ]

    def compile_one(job):
        src, extra = job
        obj = OUT_DIR / (src.name + ".o")
        cmd = [CXX] + common + extra + inc + ["-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(src.name, "ok")
        return obj

    with ThreadPoolExecutor(max_workers=4) as ex:
        objs = list(ex.map(compile_one, jobs))
    tlib = Path(torch.__file__).parent / "lib"
    cmd = [CXX, "-shared", "-o", str(lib)] + [str(o) for o in objs] + [f"-L{tlib}", f"-Wl,-rpath,{tlib}", "-lc10", "-ltorch",
                                                                        "-ltorch_cpu", "-ltorch_python", "-fopenmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    for o in objs:
        o.unlink()
    stamp.write_text(want)
    return lib


def load_ref():
    """Import oracle/_ref/esac_ref (building it first when the reference sources are present).  Returns None if it is
    neither built nor buildable."""
    lib = build_ref()
    if lib is None or not lib.exists():
        return None
    import importlib.util
    import cv2  # noqa: F401  the shim imports it
    import torch  # noqa: F401  libtorch must be loaded before the extension
    spec = importlib.util.spec_from_file_location("esac_ref", str(lib))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build_ref(force="--force" in sys.argv, verbose=True))
