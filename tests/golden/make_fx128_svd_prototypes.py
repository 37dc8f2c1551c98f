"""Generator of tests/golden/faer_ffi_fx128_svd_prototypes.json: the prototypes the reference's `faer-ffi/faer.h` declares for the
double-double kinds (fx128 / cx128) of the `svd` family, with the parser of make_ffi_prototypes.py. Run where the
reference is present: python tests/golden/make_fx128_svd_prototypes.py. tests/test_fx128_svd_cabi_cpu.py compares
include/faer_b200_fx128_svd.h with it."""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_ffi_prototypes import REF, ROOT, prototypes  # noqa: E402

FAMILY = r"^libfaer_v0_23_(BidiagParams|SvdParams|svd(_scratch)?)_(fx128|cx128)$"


def main() -> int:
    ref = prototypes(open(REF).read())
    doc = {
        "source": "faer-ffi/faer.h (reference), parsed by tests/golden/make_fx128_svd_prototypes.py",
        "prototypes": {n: ref[n] for n in sorted(ref) if re.match(FAMILY, n)},
    }
    json.dump(doc, open(os.path.join(ROOT, "tests", "golden", "faer_ffi_fx128_svd_prototypes.json"), "w"), indent=0, sort_keys=True)
    print(len(doc["prototypes"]), "prototypes written")
    return 0


if __name__ == "__main__":
    sys.exit(main())
