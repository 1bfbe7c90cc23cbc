#!/bin/sh
# Regenerates the golden GAF files of the GAF output options (tests/gafcases.py) from the UNMODIFIED reference
# (oracle/_ref/minigraph, built by oracle/Makefile), like make_golden.sh does for the plain `-c` runs.
set -e
cd "$(dirname "$0")/../.."
R=oracle/_ref/minigraph; S=tools/mgsim; G=tests/golden; F=$G/fixtures
# GAF output options (--secondary, --show-unmap, -S, --write-mz, --vc, --no-comp-path, no -c, read pairs, stable-sequence paths):
# the c3 SV-graph reads plus the edge reads of fixtures/edge.fa; read pairs in two files; reads on the hand-written rGFA
# fixtures/stable.gfa (segments without SN, a stable sequence with an SO gap, SR > 0 with min > 0, a reverse-complemented repeat)
T=$(mktemp -d)
X="--secondary=yes --show-unmap=yes -S --write-mz"
$S graph -l 300000 -n 3 -s 7 -o $T/sv 2>/dev/null
$S reads -i $T/sv.hap.fa -n 24 -l 15000 -e ont -s 5 -o $T/sv.reads.fa 2>/dev/null
cat $T/sv.reads.fa $F/edge.fa > $T/sve.fa
$R -cx lr $X $T/sv.gfa $T/sve.fa 2>/dev/null | gzip -n9 > $G/f1_sv_edge.lr.2nd_unmap_S_mz.gaf.gz
$R -cx lr $X --vc $T/sv.gfa $T/sve.fa 2>/dev/null | gzip -n9 > $G/f2_sv_edge.lr.2nd_unmap_S_mz_vc.gaf.gz
$R -cx lr $X --no-comp-path $T/sv.gfa $T/sve.fa 2>/dev/null | gzip -n9 > $G/f3_sv_edge.lr.2nd_unmap_S_mz_nocomp.gaf.gz
$R -x lr $X $T/sv.gfa $T/sve.fa 2>/dev/null > $G/f4_sv_edge.lr_nocigar.2nd_unmap_S_mz.gaf
$S walk -g $F/MT.gfa -w ">MTh0>MTh4001>MTh4502>MTh9505>MTh13014>MTh13516" -w ">MTh0<MTo3426>MTh4502>MTo8961>MTh9505>MTh13516" -o $T/mt.hap.fa
$S reads -i $T/mt.hap.fa -n 60 -l 500 -e hifi -s 61 -o $T/mt.sr.fa 2>/dev/null
python3 tests/gafcases.py pairs $T/mt.sr.fa $T/r1.fa $T/r2.fa
$R -x sr --show-unmap=yes $F/MT.gfa $T/r1.fa $T/r2.fa 2>/dev/null > $G/f5_MT_60pairs_hifi_s61.sr.gaf
$S walk -g $F/stable.gfa -w ">s1>s2>s3" -w ">s1>s4>s3" -w ">s1>s5>s3" -o $T/st.hap.fa
$S reads -i $T/st.hap.fa -n 40 -l 2500 -e hifi -s 17 -o $T/st.reads.fa 2>/dev/null
$R -cx lr $X $F/stable.gfa $T/st.reads.fa 2>/dev/null > $G/f6_stable_40x2500_hifi_s17.lr.2nd_unmap_S_mz.gaf
$R -cx lr $X --no-comp-path $F/stable.gfa $T/st.reads.fa 2>/dev/null > $G/f7_stable_40x2500_hifi_s17.lr.2nd_unmap_S_mz_nocomp.gaf
rm -rf $T
md5sum $G/f*.gaf; ls -la $G/f*.gz
