"""Every kernel launch of the product goes through cilantro_b200/csrc/launch.cuh, which counts it in kernel_launches and
checks it at once. A launch written anywhere else would be uncounted or unchecked, so the sources may not hold one."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cilantro_b200", "csrc")

RULES = {
    "<<< launch": re.compile(r"<<<"),
    "runtime launch call": re.compile(r"\bcudaLaunch(KernelEx|CooperativeKernel)\b"),
    "write to the launch counter": re.compile(r"\blaunches\s*(\+=|\+\+)|\+\+\s*(\w+\s*(->|\.)\s*)*launches\b"),
}


def test_every_launch_goes_through_launch_cuh():
    offenders = []
    for f in sorted(os.listdir(CSRC)):
        if f == "launch.cuh" or not f.endswith((".cu", ".cuh", ".hpp", ".h", ".cpp")):
            continue
        with open(os.path.join(CSRC, f), errors="ignore") as fh:
            for no, line in enumerate(fh, 1):
                offenders += [f"{f}:{no}: {what}: {line.strip()}" for what, pat in RULES.items() if pat.search(line)]
    assert not offenders, "\n".join(offenders)


def test_launch_cuh_holds_the_rules():
    with open(os.path.join(CSRC, "launch.cuh")) as fh:
        text = fh.read()
    for what, pat in RULES.items():
        assert pat.search(text), what
