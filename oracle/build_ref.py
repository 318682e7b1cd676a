#!/usr/bin/env python
"""Build the REFERENCE's own native NMS into oracle/_ref/ (test infrastructure only).

TEST INFRASTRUCTURE -- never imported by the product path.

What it does
------------
Compiles /root/reference/models/cpu_nms.pyx (the live NMS of the reference,
models/proposal_layer.py:176-178 and forward.py:54) from where it lies, with
Cython + gcc, into ``oracle/_ref/ref_cpu_nms*.so``.  The reference file cannot
be cythonized unmodified on NumPy 2 (SURVEY.md Q14: ``np.int_t`` no longer
exists in NumPy's pxd, ``np.int``/``np.float`` aliases are gone), so a
3-token (two-pattern) alias substitution is applied *in a temp dir at build time*:

    np.int_t   -> np.intp_t      (cpu_nms.pyx:26,29  -- index dtype only)
    dtype=np.int -> dtype=np.intp (cpu_nms.pyx:30    -- index dtype only)

The arithmetic lines (cpu_nms.pyx:44-67) are untouched.  ``np.float thresh``
(cpu_nms.pyx:18) is left exactly as written: Cython 3 binds it as a Python
object argument, so ``ovr >= thresh`` is a *double* comparison of the
float32-valued ``ovr`` against the Python float -- the semantics SURVEY.md Q4
records (checked in the generated C: PyFloat_FromDouble(ovr) then a float
rich-compare).

No reference source is copied into the repository: the patched text only ever
exists under a temporary directory, and only the compiled ``.so`` lands in
``oracle/_ref/`` (git-ignored build product).

``build_bbox()`` / ``load_bbox()`` do the same for models/bbox.pyx (``bbox_overlaps``, the IoU matrix of
the training path, anchor_target_layer.py:181-185) into ``oracle/_ref/ref_bbox*.so``; its alias patch is

    DTYPE = np.float -> DTYPE = np.float64   (bbox.pyx:12)
    np.float_t       -> np.float64_t         (bbox.pyx:13; the same C double)

If the reference checkout is absent this script is a no-op and the
pre-built ``.so`` -- if any -- is used as is.
"""
import os
import subprocess
import sys
import sysconfig
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = os.environ.get("FRCNN_REFERENCE_ROOT", "/root/reference")


def _patched_pyx(src_text):
    n_int_t = src_text.count("np.int_t")
    txt = src_text.replace("np.int_t", "np.intp_t")
    n_int = txt.count("dtype=np.int)")
    txt = txt.replace("dtype=np.int)", "dtype=np.intp)")
    assert n_int_t == 2 and n_int == 1, (n_int_t, n_int)
    return txt


def _patched_bbox_pyx(src_text):
    n_a = src_text.count("DTYPE = np.float\n")
    txt = src_text.replace("DTYPE = np.float\n", "DTYPE = np.float64\n")
    n_b = txt.count("np.float_t")
    txt = txt.replace("np.float_t", "np.float64_t")
    assert n_a == 1 and n_b == 1, (n_a, n_b)
    return txt


def build(verbose=False):
    """Returns the path of the built cpu_nms module, or None if the reference is absent."""
    return _build_module("cpu_nms", _patched_pyx, verbose)


def build_bbox(verbose=False):
    """Returns the path of the built bbox (bbox_overlaps) module, or None if the reference is absent."""
    return _build_module("bbox", _patched_bbox_pyx, verbose)


def _build_module(stem, patch, verbose=False):
    src = os.path.join(REF, "models", stem + ".pyx")
    os.makedirs(OUT, exist_ok=True)
    ext_suffix = sysconfig.get_config_var("EXT_SUFFIX")
    target = os.path.join(OUT, "ref_" + stem + ext_suffix)
    if not os.path.exists(src):
        return target if os.path.exists(target) else None
    if os.path.exists(target) and os.path.getmtime(target) >= os.path.getmtime(src) \
            and os.path.getmtime(target) >= os.path.getmtime(__file__):
        return target
    import numpy as np
    with tempfile.TemporaryDirectory(prefix="frcnn_ref_") as tmp:
        with open(src) as f:
            txt = patch(f.read())
        pyx = os.path.join(tmp, "ref_%s.pyx" % stem)
        with open(pyx, "w") as f:
            f.write(txt)
        c_file = os.path.join(tmp, "ref_%s.c" % stem)
        subprocess.check_call([sys.executable, "-m", "cython", "-3", pyx, "-o", c_file],
                              stdout=None if verbose else subprocess.DEVNULL)
        inc = sysconfig.get_paths()["include"]
        cmd = ["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-w",
               "-I", inc, "-I", np.get_include(), c_file, "-o", target]
        subprocess.check_call(cmd)
    return target


def load():
    """Import the compiled reference NMS; returns the module or None."""
    return _load("ref_cpu_nms", build())


def load_bbox():
    """Import the compiled reference bbox_overlaps; returns the module or None."""
    return _load("ref_bbox", build_bbox())


def _load(name, path):
    if path is None or not os.path.exists(path):
        return None
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print("oracle/_ref:", build(verbose=True))
    print("oracle/_ref:", build_bbox(verbose=True))
