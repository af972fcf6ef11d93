"""Install the reference into baseline/_ref (git-ignored).

1. the prescribed offline pip install — fails: the reference has no setup.py/pyproject.toml
   ("Directory ... is not installable");
2. fallback: verbatim copy of the main-tree sources (server.py, client.py, config.yaml, src/)
   with a sha256 manifest so the harness can prove the copy is unmodified.
"""
import hashlib
import json
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = os.environ.get("SLB200_REFERENCE_DIR", "")   # checkout of the reference repository
DST = os.path.join(HERE, "_ref")


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def install(force=False):
    if os.path.exists(os.path.join(DST, "MANIFEST.json")) and not force:
        return DST
    if not REF_SRC or not os.path.isdir(REF_SRC):
        raise RuntimeError("set SLB200_REFERENCE_DIR to a checkout of the reference repository")
    tmp = "/tmp/_slb200_refcopy"
    shutil.rmtree(tmp, ignore_errors=True)
    shutil.copytree(REF_SRC, tmp, ignore=shutil.ignore_patterns(".git", "other", "pics"))
    pip = subprocess.run([sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--find-links",
                          "/opt/wheelhouse", "--target", DST, tmp], capture_output=True, text=True)
    outcome = "pip install ok" if pip.returncode == 0 else "pip: " + (pip.stderr.strip().splitlines() or ["failed"])[-1]
    if pip.returncode != 0:
        shutil.rmtree(DST, ignore_errors=True)
        shutil.copytree(tmp, DST)
    manifest = {"outcome": outcome, "files": {}}
    for root, _, files in os.walk(DST):
        for fn in files:
            if fn.endswith((".py", ".yaml")):
                p = os.path.join(root, fn)
                rel = os.path.relpath(p, DST)
                src = os.path.join(REF_SRC, rel)
                manifest["files"][rel] = {"sha256": _sha(p), "matches_reference": os.path.exists(src) and _sha(src) == _sha(p)}
    with open(os.path.join(DST, "MANIFEST.json"), "w") as f:
        json.dump(manifest, f, indent=1)
    return DST


if __name__ == "__main__":
    d = install(force="--force" in sys.argv)
    m = json.load(open(os.path.join(d, "MANIFEST.json")))
    print(d, m["outcome"], "files:", len(m["files"]), "all match:", all(v["matches_reference"] for v in m["files"].values()))
