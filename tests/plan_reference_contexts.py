"""Build plans hand-written after the Dockerfiles of two of the reference's build contexts
(testdata/build-context/copy-glob and copy-from, stored in tests/golden/reference_testdata.tar.gz), and the generator
of their pinned cacheIDs, tests/golden/plan_cache_ids.json:
    python -m tests.plan_reference_contexts"""
import json
import os
import tarfile
import tempfile

from makisu_b200.host import PlanStep
from oracle import ctx_crc
from tests import plan_oracle

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "plan_cache_ids.json")

RUN, COPY = "RUN", "COPY"
PLANS = {
    "copy-glob": [
        PlanStep.from_image("debian:8"),
        PlanStep.copy(COPY, "*.json /", ["*.json"]),
        PlanStep.base(RUN, "cat /1.json", False),
        PlanStep.from_image("debian:8"),
        PlanStep.base(RUN, "mkdir /mine", False),
        PlanStep.copy(COPY, "--from=phase1 /*.json /mine/", ["/*.json"], from_stage="phase1"),
        PlanStep.copy(COPY, "*.txt /mine/", ["*.txt"]),
        PlanStep.base(RUN, "cat /mine/1.txt", False),
        PlanStep.base("ENTRYPOINT", '["/bin/sh", "-c", "ls /"]', False),
    ],
    "copy-from": [
        PlanStep.from_image("busybox:latest"),
        PlanStep.base(RUN, 'echo "OK" > /test1.txt', False),
        PlanStep.from_image("busybox:latest"),
        PlanStep.copy(COPY, "--from=0 /test1.txt /test2.txt", ["/test1.txt"], from_stage="0"),
        PlanStep.base(RUN, "cat /test2.txt", False),
        PlanStep.from_image("debian:8", remote=True),
        PlanStep.from_image("busybox"),
        PlanStep.copy(COPY, "--from=debian:8 /bin/bash /bash", ["/bin/bash"], from_stage="debian:8"),
        PlanStep.base(RUN, "ls -la /bash", False),
        PlanStep.from_image("alpine"),
        PlanStep.base(RUN, "mkdir /dst", False),
        PlanStep.copy(COPY, "--chown=ftp:ftp 1/ /dst/d/", ["1/"]),
        PlanStep.copy(COPY, "--chown=ftp:ftp 1/ /dst/dst/d", ["1/"]),
        PlanStep.copy(COPY, ". /all/", ["."]),
        PlanStep.base(RUN, "cat /dst/d/1.txt", True),
    ],
}
SEED = ctx_crc.plan_seed(False, True)


def unpack(dst: str) -> str:
    """The reference's build-context tree under dst; returns its path."""
    with tarfile.open(os.path.join(HERE, "golden", "reference_testdata.tar.gz")) as tf:
        tf.extractall(dst, filter="data")
    return os.path.join(dst, "build-context")


def main():
    with tempfile.TemporaryDirectory() as d:
        root = unpack(d)
        out = {"seed": SEED, "plans": {k: plan_oracle.plan_cache_ids(SEED, os.path.join(root, k), v) for k, v in PLANS.items()}}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
