"""Generator of tests/golden/full_piv_lu_gh238.json: the 28 x 28 matrix and the right-hand side of the reference's
`test_gh238` (faer/src/linalg/lu/full_pivoting/factor.rs, fn test_gh238), whose full-pivoting solve must be all finite.
Run in the build container (the reference is not present on the GPU box): python tests/golden/make_full_piv_lu_fixture.py"""
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = "/root/reference/faer/src/linalg/lu/full_pivoting/factor.rs"


def _numbers(block: str):
    return [float(x) for x in re.findall(r"-?\d+\.\d*(?:e-?\d+)?", block)]


def main() -> int:
    src = open(REF).read()
    body = src[src.index("fn test_gh238"):]
    a_blk = body[body.index("let A = ["):body.index("];")]
    b_start = body.index("let b = [")
    b_blk = body[b_start:body.index("];", b_start)]
    A = _numbers(a_blk)
    b = _numbers(b_blk)
    n = int(round(len(A) ** 0.5))
    assert n * n == len(A) and len(b) == n, (len(A), len(b))
    doc = {"source": "faer/src/linalg/lu/full_pivoting/factor.rs (reference), fn test_gh238; A is row-major",
           "n": n, "A_row_major": A, "b": b}
    json.dump(doc, open(os.path.join(ROOT, "tests", "golden", "full_piv_lu_gh238.json"), "w"), indent=0)
    print(f"gh238: {n} x {n}, rhs of {len(b)}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
