"""CPU test: every environment variable the library reads is documented, and every documented one is read.

The names are collected from the sources: the `getenv("FAER_B200_...")` literals under csrc/ and the environment names of
the run-time options in runtime.cu's `g_opt_defs`. They must be exactly the names in INTEGRATION.md's "Run-time knobs"
table, so a switch cannot be added without documenting it, nor removed while the table still offers it."""
import glob
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "faer-rs_b200", "csrc")


def _names_read_by_csrc():
    names = set()
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))):
        with open(path, encoding="utf-8") as f:
            names.update(re.findall(r'getenv\(\s*"(FAER_B200_\w+)"\s*\)', f.read()))
    with open(os.path.join(CSRC, "runtime.cu"), encoding="utf-8") as f:
        defs = re.search(r"g_opt_defs\[OPT_COUNT\]\s*=\s*\{(.*?)\};", f.read(), re.S)
    assert defs, "runtime.cu: g_opt_defs not found"
    opt_names = re.findall(r'"(FAER_B200_\w+)"', defs.group(1))
    assert opt_names, "runtime.cu: g_opt_defs names no environment variable"
    names.update(opt_names)
    return names


def _names_in_knob_table():
    with open(os.path.join(ROOT, "INTEGRATION.md"), encoding="utf-8") as f:
        text = f.read()
    section = re.search(r"^## Run-time knobs[^\n]*\n(.*?)(?=^## |\Z)", text, re.S | re.M)
    assert section, "INTEGRATION.md: no 'Run-time knobs' section"
    names = set()
    for line in section.group(1).splitlines():
        if line.startswith("|"):
            names.update(re.findall(r"`(FAER_B200_\w+)`", line.split("|")[1]))
    return names


def test_knob_table_lists_exactly_the_variables_the_library_reads():
    read, documented = _names_read_by_csrc(), _names_in_knob_table()
    assert read, "no FAER_B200_* variable found under csrc/"
    assert read - documented == set(), "read by csrc/ but missing from INTEGRATION.md's knob table"
    assert documented - read == set(), "in INTEGRATION.md's knob table but read nowhere in csrc/"
