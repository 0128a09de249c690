#!/usr/bin/env bash
# SASS listings of the hot kernels -> profiles/sass/*.sass (git-ignored) (encodings stripped; -lineinfo comments kept).  No GPU needed:
#   python -m aerial_gym_simulator_b200._build --force && bash tools/dump_sass.sh
# What to look for: UBLKCP + SYNCS (1-D TMA bulk copy on an mbarrier) in hp2_cast_kernel_smem_tile; ACQBULK-free persistent loop;
# MEMBAR.SC.SYS / ST.E.STRONG.SYS (system-scope fence + release store of the flag) in obs_gather_push_kernel; REDG / ATOMG on the
# tile counters and no CALL in hp1_step_kernel_*.
set -eu
cd "$(dirname "$0")/../aerial_gym_simulator_b200/build"
out=../../profiles/sass
mkdir -p $out
for spec in "hp1.o:hp1_step_kernelILi4ELb1ELb1ELi241E:hp1_step_kernel_4_task_coop_spec241" \
            "hp2_raycast.o:hp2_cast_kernelILb1ELb1E:hp2_cast_kernel_smem_tile" \
            "hp2_raycast.o:hp2_cast_kernelILb0ELb1E:hp2_cast_kernel_records_tile" \
            "p2p_allgather.o:obs_gather_push_kernel:obs_gather_push_kernel"; do
  o=${spec%%:*}; rest=${spec#*:}; pat=${rest%%:*}; name=${rest#*:}
  cuobjdump -sass $o | awk -v pat="$pat" '/Function :/{p=index($0,pat)>0} p' | sed -E 's#/\* 0x[0-9a-f]+ \*/##; s/[[:space:]]+$//' | grep -v "^\s*$" > $out/$name.sass
  echo "$name: $(grep -c '^\s*/\*[0-9a-f]\{4,5\}\*/' $out/$name.sass) instructions"
done
