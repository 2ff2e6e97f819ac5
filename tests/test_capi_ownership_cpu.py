"""Every device allocation, pinned buffer, event and stream of the C ABI has an owner (capi.cu: DevPtr, PinnedPtr, Event,
Stream).  Their deleters are the only places that release such a resource, so a function that returns early on a failed
CUDA call (CU) leaves nothing behind.  A hand-written release elsewhere in the file means a resource without an owner."""
from __future__ import annotations

import os
import re

from tests.util import ROOT

CAPI = os.path.join(ROOT, "circom_b200", "csrc", "capi.cu")
RELEASES = ("cudaFree", "cudaFreeHost", "cudaEventDestroy", "cudaStreamDestroy")
# the one-line deleters of the owning types
DELETER = re.compile(r"^struct \w+ \{ void operator\(\)\((void \*|cudaEvent_t |cudaStream_t )\w+\) const \{ (\w+)\(\w+\); \} \};$")


def test_resources_are_released_only_by_their_owners():
    calls = []
    for no, line in enumerate(open(CAPI).read().splitlines(), 1):
        for name in re.findall(r"\b(%s)\s*\(" % "|".join(RELEASES), line):
            calls.append((no, name, line.strip()))
    outside = [(no, line) for no, name, line in calls if not (DELETER.match(line) and DELETER.match(line).group(2) == name)]
    assert outside == [], "resources released outside the owning types (capi.cu line, text): %s" % outside
    assert sorted(name for _, name, _ in calls) == sorted(RELEASES), "one deleter per kind of resource"
