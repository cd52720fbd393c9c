"""Fixture for tests/test_boundary_cpu.py: the (reference file, name) pairs of tests/standins.CONTRACT that occur, as whole words, in
the UNMODIFIED reference file they are cited from.  Only names found there are written, so a contract name the reference does not
define makes the test fail until it is removed from the contract (or the fixture is regenerated against a reference that has it).

  python tests/golden/make_golden_contract.py     (needs the reference tree; writes tests/golden/contract_names.json)
"""
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)


def main():
    from oracle.refshim.load_reference import REFERENCE_ROOT
    from tests.standins import CONTRACT
    found, missing = {}, []
    for side in CONTRACT.values():
        for rel, names in side.items():
            src = open(os.path.join(REFERENCE_ROOT, rel)).read()
            for n in names:
                if re.search(r"\b" + re.escape(n) + r"\b", src):
                    found.setdefault(rel, set()).add(n)
                else:
                    missing.append((rel, n))
    with open(os.path.join(HERE, "contract_names.json"), "w") as f:
        json.dump({rel: sorted(v) for rel, v in sorted(found.items())}, f, indent=1, sort_keys=True)
        f.write("\n")
    print(sum(len(v) for v in found.values()), "pairs found;", "missing:", missing)


if __name__ == "__main__":
    main()
