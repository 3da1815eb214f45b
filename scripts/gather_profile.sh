#!/bin/sh
# Gather profile of the multi-commit kernel on C4 (one H100): scripts/round_profile.sh with a -DMULTI_GATHER_PROFILE library instead.
# Prints CTA 0's split of the gather ("Gather profile" in csrc/ccsim_multi.cuh) and the publish skew over all CTAs per wave.
PROFILE_DEFINE=-DMULTI_GATHER_PROFILE exec "$(dirname "$0")/round_profile.sh" "$@"
