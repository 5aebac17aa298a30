#!/usr/bin/env python
"""Fingerprints of the device code that HAS run on an H100 (docs/sass/VALIDATED.sha256).

The contract for work around GPU-validated kernels (shared headers, policy templates, new variants next to them) is:
the instructions of a validated kernel do not change unless it is re-validated on a GPU.  This tool makes that
checkable without a GPU:

  python scripts/sass_fingerprint.py            compare build/kernels/*.o with the manifest (exit 1 on a mismatch)
  python scripts/sass_fingerprint.py --write [--baseline DIR]
                                                rewrite the manifest from the current objects after a GPU re-validation;
                                                with --baseline (a directory of kernel objects built from the commit
                                                that ran on the GPU) only functions that have a byte-identical twin
                                                there are listed

A fingerprint is the first 64 bits (16 hex digits) of the SHA-256 of a function's SASS instruction stream (addresses
and encodings included, the path-dependent anonymous-namespace tag of the symbol name normalised).  Functions that
have NOT run on a GPU yet are listed in UNVALIDATED below and are left out of the manifest.
"""
import hashlib
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MANIFEST = os.path.join(ROOT, "docs", "sass", "VALIDATED.sha256")
# demangled-name patterns of instantiations that only a run with several GPUs launches (the suite's one-GPU run emulates
# at most the rank counts below on one device)
UNVALIDATED = (
    # more than 8 ranks: needs > 8 GPUs (ranks sharing one GPU's hardware queue serialise their spinning kernels)
    r"two_shot_kernel<[\w ]+, 16, 1>",
)


def functions(obj):
    text = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    out, name = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name is not None and re.match(r"\s+/\*[0-9a-f]{4}\*/|\s+/\* 0x", line):
            out[name].append(" ".join(line.split()))  # cuobjdump pads columns to the widest line of the FILE
    return out


def demangle(names):
    p = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True)
    clean = [re.sub(r"\(anonymous namespace\)::|hpcp::|^void ", "", d).split("(")[0] for d in p.stdout.splitlines()]
    return dict(zip(names, clean))


def current():
    subprocess.run(["make", "-s", "build/libhpcp.a"], cwd=ROOT, check=True, stdout=subprocess.DEVNULL)
    rows = {}
    kdir = os.path.join(ROOT, "build", "kernels")
    for obj in sorted(os.listdir(kdir)):
        if not obj.endswith(".o"):
            continue
        fns = functions(os.path.join(kdir, obj))
        names = demangle(list(fns))
        for mangled, lines in fns.items():
            d = names[mangled]
            if any(re.search(pat, d) for pat in UNVALIDATED):
                continue
            rows[f"{obj[:-2]}::{d}"] = hashlib.sha256("\n".join(lines).encode()).hexdigest()[:16]
    return rows


def main(argv):
    rows = current()
    if "--write" in argv:
        if "--baseline" in argv:
            kdir = argv[argv.index("--baseline") + 1]
            base = set()
            for obj in os.listdir(kdir):
                if obj.endswith(".o"):
                    base |= {hashlib.sha256("\n".join(v).encode()).hexdigest()[:16]
                             for v in functions(os.path.join(kdir, obj)).values()}
            rows = {k: h for k, h in rows.items() if h in base}
        header = []
        if os.path.exists(MANIFEST):  # keep the explanatory header
            header = [line for line in open(MANIFEST) if line.startswith("#")]
        with open(MANIFEST, "w") as f:
            f.writelines(header or ["# sha256 of the SASS of every kernel that has run on an H100 "
                                    "(scripts/sass_fingerprint.py)\n"])
            for k in sorted(rows):
                f.write(f"{rows[k]}  {k}\n")
        print(f"wrote {len(rows)} fingerprints to {os.path.relpath(MANIFEST, ROOT)}")
        return 0
    want = {}
    with open(MANIFEST) as f:
        for line in f:
            if line.strip() and not line.startswith("#"):
                h, k = line.split(None, 1)
                want[k.strip()] = h
    bad = [k for k in want if rows.get(k) != want[k]]
    for k in bad:
        print(("CHANGED  " if k in rows else "MISSING  ") + k)
    print(f"{len(want) - len(bad)} of {len(want)} validated kernels are byte-identical")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
