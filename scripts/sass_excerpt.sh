#!/usr/bin/env bash
# SASS evidence from the built library (no GPU needed): which instructions the scan kernels are made of.
LIB=toppra_b200/libtoppra_b200.so
cuobjdump -sass $LIB > /tmp/tb_lib.sass 2>/dev/null
echo "# $LIB  ($(cuobjdump -lelf $LIB | grep -c sm_90a) sm_90a cubin(s), $(grep -c 'Function :' /tmp/tb_lib.sass) kernels)"
echo "# mnemonic counts over all kernels"
for op in UBLKCP SYNCS.ARRIVE SYNCS.PHASECHK REDUX SHFL.IDX SHFL.BFLY VOTE MUFU.RCP64H MUFU.RSQ64H DFMA DADD DMUL DSETP ELECT HMMA UTCHMMA; do
  printf "%-16s %s\n" "$op" "$(grep -c "$op" /tmp/tb_lib.sass)"
done
echo "# (DFMA in a -fmad=false build: only inside the IEEE division / sqrt / sincos sequences; no tensor-core instructions: there is no dense contraction)"
echo
echo "# record scan scan_kernel<1,1,32,false,0,false,false>: bulk copy of a stage record + mbarrier wait + redux reductions"
awk '/Function :/ {f = (index($0, "scan_kernelILi1ELi1ELi32ELb0ELi0ELb0ELb0E") > 0)} f' /tmp/tb_lib.sass | grep -E "UBLKCP|SYNCS|REDUX|ELECT" | head -16 | sed -E 's/ +\/\* 0x[0-9a-f]+ \*\///' | cut -c1-110
echo
echo "# fused scan scan_kernel<1,1,28,false,0,true,false> (tb_scan_velacc): no bulk copies (rows are built from the spline), redux + shuffles"
awk '/Function :/ {f = (index($0, "scan_kernelILi1ELi1ELi28ELb0ELi0ELb1ELb0E") > 0)} f' /tmp/tb_lib.sass | grep -E "REDUX|SHFL|MUFU.RCP64H|LDS.128" | head -14 | sed -E 's/ +\/\* 0x[0-9a-f]+ \*\///' | cut -c1-110
echo
echo "# static size of the scan instantiations (instructions / S2R / LDL / STL / REDUX / SHFL / RCP64H)"
for k in ILi1ELi1ELi28ELb0ELi0ELb1ELb0E ILi1ELi1ELi32ELb0ELi0ELb1ELb0E ILi1ELi1ELi32ELb0ELi0ELb0ELb0E ILi2ELi1ELi20ELb0ELin1ELb0ELb0E; do
  printf "%-36s " "scan_kernel<$k>"; scripts/sass_stats.sh $k toppra_b200/csrc/tb_scan.o
done
