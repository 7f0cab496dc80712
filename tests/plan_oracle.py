"""ORACLE (test infrastructure only): the cacheIDs of a whole build plan, chained from the per-step restatements of
oracle/ctx_crc.py the way processStagesAndAliases and createDockerfileSteps chain them
(reference lib/builder/build_plan.go:93-160, build_stage.go:78-108,153-165): every step is seeded with the cacheID of
the step before it, except that a remote-image stage inserted for a COPY --from (build_plan.go:142-152) was created
after the stage that names it had already taken its seed -- so a run of such stages chains from that seed and the stage
after the run takes the same seed again.

Steps are anything with the attributes of makisu_b200.host.PlanStep (kind, directive, args, from_paths, from_stage,
commit)."""
from __future__ import annotations

from typing import List, Sequence

from oracle import ctx_crc

STEP_COPY, STEP_FROM, STEP_BASE, STEP_REMOTE_FROM = 1, 2, 3, 4  # include/mkhost.h MKHOST_STEP_*


def plan_cache_ids(seed: str, context_dir: str, steps: Sequence) -> List[str]:
    ids: List[str] = []
    sd, stage_seed, in_remote = seed, seed, False
    for s in steps:
        remote = s.kind == STEP_REMOTE_FROM
        if remote and not in_remote:
            stage_seed = sd
        elif not remote and in_remote:
            sd = stage_seed
        in_remote = remote
        if s.kind in (STEP_FROM, STEP_REMOTE_FROM):
            cid = ctx_crc.from_step_cache_id(sd, s.args)
        elif s.kind == STEP_BASE:
            cid = ctx_crc.base_step_cache_id(sd, s.directive, s.args, bool(s.commit))
        elif s.kind == STEP_COPY:
            cid = ctx_crc.copy_step_cache_id(sd, s.directive, s.args, context_dir, list(s.from_paths), s.from_stage)
        else:
            raise ValueError("unknown step kind %r" % s.kind)
        ids.append(cid)
        sd = cid
    return ids


def unique_file_bytes(context_dir: str, steps: Sequence) -> int:
    """Bytes of the distinct regular files the COPY/ADD steps of a plan hash (each file once)."""
    seen = {}
    for s in steps:
        if s.kind == STEP_COPY and not s.from_stage:
            for seg in ctx_crc.context_segments(context_dir, list(s.from_paths)):
                if seg.kind == "file":
                    seen[seg.path] = seg.size
    return sum(seen.values())
