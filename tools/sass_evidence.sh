#!/bin/bash
# dev tool: SASS evidence of the tensor-core / TMA / mbarrier paths in the shipped library
LIB=${1:-a1-qp-mpc-controller_b200/liba1mpc.so}
echo "# cuobjdump -sass $LIB  ($(date -u +%Y-%m-%d), $(nvcc --version | grep release | sed 's/.*release //'))"
echo "# per kernel: count of DMMA.8x8x4 (fp64 tensor-core MMA), UBLKCP (cp.async.bulk TMA copy), SYNCS.* (mbarrier arrive / try_wait), DFMA"
cuobjdump -sass "$LIB" | awk '
/Function :/ { f=$3 }
/DMMA/ { d[f]++ } /UBLKCP/ { u[f]++ } /SYNCS/ { s[f]++ } /DFMA/ { m[f]++ } /MUFU.RSQ64H/ { r[f]++ }
END { for (k in m) printf "%6d DMMA %2d UBLKCP %3d SYNCS %6d DFMA %3d MUFU.RSQ64H  %s\n", d[k]+0, u[k]+0, s[k]+0, m[k], r[k]+0, k }' | sort -k1,1nr | while read -r line; do n=$(echo "$line" | awk '{print $NF}'); echo "$(echo "$line" | sed "s|$n||") $(echo $n | c++filt | cut -c1-110)"; done
echo
echo "# excerpt: first lines with each mnemonic in solve_kernel<2,10,8,0,0> (the trot class)"
cuobjdump -sass -fun 2>/dev/null '_ZN5a1mpc12solve_kernelILi2ELi10ELi8ELi0ELb0EEEvNS_9DevParamsEPKdPKiNS_10DevOutputsE' "$LIB" | grep -E "UBLKCP|SYNCS|DMMA|MUFU.RSQ64H" | awk '{k=$0; sub(/^[ \t]*\/\*[0-9a-f]+\*\/[ \t]*/,"",k); split(k,a," "); m=a[1]; if (m ~ /^@/) m=a[2]; sub(/\..*/,"",m); if (c[m]++ < 3) print "   " k}' | cut -c1-150
echo
echo "# warp teams: named-barrier instructions of solve_kernel<4,10,4,1,0> (four-stance class, two warps per QP): BAR.SYNC / BAR.RED with a barrier id register and 0x40 threads; ATOMG = the QP queue"
cuobjdump -sass -fun 2>/dev/null '_ZN5a1mpc12solve_kernelILi4ELi10ELi4ELi1ELb0EEEvNS_9DevParamsEPKdPKiNS_10DevOutputsE' "$LIB" | grep -E "BAR\.|ATOMG|RED\.E" | awk '{k=$0; sub(/^[ \t]*\/\*[0-9a-f]+\*\/[ \t]*/,"",k); split(k,a," "); m=a[1]; if (m ~ /^@/) m=a[2]; n[m]++; if (c[m]++ < 2) print "   " k} END { for (m in n) printf "   # %d x %s\n", n[m], m }' | cut -c1-150
