"""ORACLE build recipe (test / bench infrastructure, never imported by the product): vendor the reference's own
implementation of the path into oracle/_ref/ so that bench.py can time it on the host cores as the CPU arm.

    python oracle/build_ref.py            # reads the reference checkout at $DS_REFERENCE_ROOT; writes oracle/_ref/ only

The reference is Python: "building" it means copying the import closure of `scene_synthesis.networks`
(networks/{__init__, denoise_net, diffusion_ddpm, diffusion_scene_layout_ddpm, loss, feature_extractors,
frozen_batchnorm}.py, stats_logger.py, the package __init__) byte for byte from where the sources lie, plus empty
stand-ins for the four modules the reference imports and does not use on this path and that this image lacks
(`tkinter`, `clip`: stray IDE imports / an optional text encoder, SURVEY 8c).  oracle/_ref/ is git-ignored (history
stays free of reference sources).  Without a reference checkout build() does nothing and the bench times the oracle
port instead.  A MANIFEST with sha256 of every copied file is written
so that a run can state exactly what it timed.
"""
import hashlib
import json
import os
import shutil
import sys

SRC = os.environ.get("DS_REFERENCE_ROOT", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
DST = os.path.join(HERE, "_ref")
FILES = ["scene_synthesis/__init__.py", "scene_synthesis/stats_logger.py"] + [
    "scene_synthesis/networks/%s.py" % m for m in
    ("__init__", "denoise_net", "diffusion_ddpm", "diffusion_scene_layout_ddpm", "loss", "feature_extractors",
     "frozen_batchnorm")]
STUBS = {"tkinter/__init__.py": "", "tkinter/messagebox.py": "NO = 0\n", "tkinter/tix.py": "Tree = object\n",
         "clip/__init__.py": ""}


def build(verbose=True):
    if not os.path.isdir(SRC):
        return None                         # keep a copy vendored earlier, if any (else the bench uses the oracle port)
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    manifest = {}
    for rel in FILES:
        src, dst = os.path.join(SRC, rel), os.path.join(DST, rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(src, dst)
        manifest[rel] = hashlib.sha256(open(src, "rb").read()).hexdigest()
    for rel, body in STUBS.items():
        dst = os.path.join(DST, "_stubs", rel)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        with open(dst, "w") as f:
            f.write(body)
    with open(os.path.join(DST, "MANIFEST.json"), "w") as f:
        json.dump({"source": SRC, "files": manifest}, f, indent=1)
    if verbose:
        print("oracle/_ref: %d reference files vendored from %s" % (len(manifest), SRC))
    return DST


def activate():
    """Put the vendored reference (and its stand-in stubs, only where the real module is missing) on sys.path.
    Call in a process that has NOT imported the repo's own `scene_synthesis` shim."""
    if not os.path.isfile(os.path.join(DST, "MANIFEST.json")):
        return False
    assert "scene_synthesis" not in sys.modules, "the repo's scene_synthesis shim is already imported"
    import importlib.util
    stubs = os.path.join(DST, "_stubs")
    for name in ("tkinter", "clip"):
        if importlib.util.find_spec(name) is None and stubs not in sys.path:
            sys.path.append(stubs)
    sys.path.insert(0, DST)
    return True


if __name__ == "__main__":
    build()
