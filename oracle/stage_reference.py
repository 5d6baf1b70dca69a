"""Stage the UNMODIFIED reference (THUwangcy/ReChorus) under oracle/_ref/ for the parts of the project that run the
reference's own code: bench.py's reference arm (`--impl reference`, cpu_baseline kind "reference"), the overlay tests and
tools/run_reference.py.  oracle/_ref/ is git-ignored; build() runs this recipe, and the staged copy is what those users
read -- never the reference checkout itself.

ReChorus is a source tree without setup.py / pyproject.toml, so the recipe is a verbatim copy of its `src/` (Python only,
~580 KB).  Nothing is edited: every staged file is checked against the checkout by SHA-256 and the digests are written to
oracle/_ref/MANIFEST.json.  The checkout is found at $B2R_REFERENCE (default /root/reference); where it is absent the
recipe leaves an existing staged copy as it is and otherwise does nothing."""
import hashlib
import json
import os
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DST = os.path.join(ROOT, "oracle", "_ref")
REF_SRC = os.path.join(DST, "src")          # what the users above pass as the reference's src/ directory


def _sha(path):
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for blk in iter(lambda: f.read(1 << 20), b""):
            h.update(blk)
    return h.hexdigest()


def stage(verbose: bool = False) -> str:
    """copy <checkout>/src to oracle/_ref/src (once) and verify it; returns REF_SRC, or "" if there is nothing staged"""
    checkout = os.environ.get("B2R_REFERENCE", "/root/reference")
    if not os.path.isfile(os.path.join(checkout, "src", "main.py")):
        return REF_SRC if os.path.isfile(os.path.join(REF_SRC, "main.py")) else ""
    if not os.path.isfile(os.path.join(REF_SRC, "main.py")):
        tmp = REF_SRC + ".tmp"
        shutil.rmtree(tmp, ignore_errors=True)
        shutil.copytree(os.path.join(checkout, "src"), tmp, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        os.replace(tmp, REF_SRC)
    manifest = {}
    for base, _, files in os.walk(REF_SRC):
        if "__pycache__" in base:
            continue
        for f in sorted(files):
            p = os.path.join(base, f)
            rel = os.path.relpath(p, REF_SRC)
            manifest[rel] = _sha(p)
            orig = os.path.join(checkout, "src", rel)
            if not os.path.exists(orig) or _sha(orig) != manifest[rel]:
                raise RuntimeError(f"oracle/_ref/src/{rel} differs from the reference checkout")
    with open(os.path.join(DST, "MANIFEST.json"), "w") as f:
        json.dump({"files": manifest}, f, indent=1)
    if verbose:
        print(f"oracle/_ref: {len(manifest)} reference files staged")
    return REF_SRC


if __name__ == "__main__":
    stage(verbose=True)
