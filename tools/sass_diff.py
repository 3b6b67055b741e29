#!/usr/bin/env python
"""Per-kernel SASS fingerprint of libsptag_b200.so, and a check against a stored fingerprint.

See DESIGN.md §6: a change meant to leave device code alone (a refactor, host-only work) must leave every kernel's
instructions byte-identical, which this checks without a GPU.  The fingerprint is sha256 over the instruction lines of each
function in `cuobjdump -sass`: the instruction text and both 64-bit encoding words (so stall counts, barriers and reuse
flags count too), with the addresses stripped and the module headers between functions left out.  It is keyed by the
mangled name with the path hash of anonymous namespaces (`_GLOBAL__N__<hash>_`) removed, so
builds from different directories compare equal.

    python tools/sass_diff.py --write build/validated_sass_hashes.json     # after a validated GPU session
    python tools/sass_diff.py --check build/validated_sass_hashes.json     # after any later change
"""
import argparse
import hashlib
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "sptag_b200", "lib", "libsptag_b200.so")
INSTR = re.compile(r"\s*/\*[0-9a-f]{4,}\*/|\s*/\* 0x[0-9a-f]{16} \*/\s*$")  # an instruction (starts with its address) or its 2nd word
ANON = re.compile(r"_GLOBAL__N__[0-9a-f]+_")


def fingerprint(lib):
    txt = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    out = {}
    for part in re.split(r"\n\s*Function : ", txt)[1:]:
        name, _, body = part.partition("\n")
        ins = [re.sub(r"/\*[0-9a-f]+\*/", "", line).strip() for line in body.splitlines() if INSTR.match(line)]
        out[ANON.sub("_GLOBAL__N__", name.strip())] = hashlib.sha256("\n".join(ins).encode()).hexdigest()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=LIB)
    ap.add_argument("--write")
    ap.add_argument("--check")
    a = ap.parse_args()
    fp = fingerprint(a.lib)
    if a.write:
        with open(a.write, "w") as f:
            json.dump(fp, f, indent=0, sort_keys=True)
        print("wrote %d kernel fingerprints to %s" % (len(fp), a.write))
    if a.check:
        ref = json.load(open(a.check))
        changed = sorted(k for k in ref if fp.get(k) != ref[k])
        new = sorted(k for k in fp if k not in ref)
        print("%d stored kernels, %d changed or missing, %d new kernels" % (len(ref), len(changed), len(new)))
        for k in changed:
            print("  CHANGED", k)
        return 1 if changed else 0
    return 0


if __name__ == "__main__":
    sys.exit(main())
