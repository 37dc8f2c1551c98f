"""Generator of tests/golden/faer_ffi_evd_prototypes.json: the prototypes the reference's `faer-ffi/faer.h` declares for the
general eigendecomposition (`evd_*`, `evd_scratch_*`, `EvdParams_*`, `SchurParams_*`, `EvdFromSchurParams_*`) in f32 / f64 /
c32 / c64, and the layout of its three parameter structs, with the parser of make_ffi_prototypes.py. Run where the reference
is present: python tests/golden/make_evd_prototypes.py. tests/test_evd_cabi_cpu.py compares include/faer_b200_evd.h with it."""
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_ffi_prototypes import REF, ROOT, prototypes  # noqa: E402

FAMILY = r"^libfaer_v0_23_(evd|evd_scratch|EvdParams|SchurParams|EvdFromSchurParams)_(f32|f64|c32|c64)$"


def struct_fields(text: str, name: str) -> list:
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), text, re.S).group(1)
    return [re.sub(r"\s+", " ", f).strip() for f in body.split(";") if f.strip()]


def main() -> int:
    text = open(REF).read()
    ref = prototypes(text)
    doc = {
        "source": "faer-ffi/faer.h (reference), parsed by tests/golden/make_evd_prototypes.py",
        "prototypes": {n: ref[n] for n in sorted(ref) if re.match(FAMILY, n)},
        "structs": {s: struct_fields(text, "FaerV0_24_" + s) for s in ("EvdFromSchurParams", "SchurParams", "EvdParams")},
    }
    json.dump(doc, open(os.path.join(ROOT, "tests", "golden", "faer_ffi_evd_prototypes.json"), "w"), indent=0, sort_keys=True)
    print(len(doc["prototypes"]), "prototypes written")
    return 0


if __name__ == "__main__":
    sys.exit(main())
