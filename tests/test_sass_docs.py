"""The committed SASS evidence (docs/sass/) must describe the kernels the tree builds right now."""
import filecmp
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sass_listings_are_in_sync_with_the_sources(tmp_path):
    out = tmp_path / "sass"
    p = subprocess.run(["bash", os.path.join(ROOT, "scripts", "make_sass.sh"), str(out)], cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout + p.stderr
    committed = os.path.join(ROOT, "docs", "sass")
    assert sorted(f for f in os.listdir(out) if f.endswith(".sass")) == sorted(
        os.path.basename(o)[:-2] + ".sass" for o in os.listdir(os.path.join(ROOT, "build", "kernels")) if o.endswith(".o"))
    assert filecmp.cmp(os.path.join(out, "SUMMARY.md"), os.path.join(committed, "SUMMARY.md"), shallow=False), \
        "regenerate with scripts/make_sass.sh"
    summary = open(os.path.join(committed, "SUMMARY.md")).read()
    for mnemonic in ("HGMMA", "UTMALDG.2D", "UTMALDG.2D.MULTICAST", "UBLKCP", "LDGMC", "UTMAREDG.2D.ADD",
                     "REDG.E.ADD.F32x4"):
        assert mnemonic in summary, mnemonic


def test_kernels_that_ran_on_a_gpu_are_byte_identical():
    """docs/sass/VALIDATED.sha256 lists the SASS fingerprints of the kernels as they ran on an H100; refactors around
    them (shared headers, policy templates, new variants) must not change a single instruction."""
    import sys

    p = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "sass_fingerprint.py")], cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "validated kernels are byte-identical" in p.stdout
