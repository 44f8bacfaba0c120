#!/bin/bash
# Counts the SASS mnemonics that show what the kernels of libesac_b200.so are built from (UBLKCP / SYNCS = TMA bulk copy +
# mbarrier, LDGSTS = cp.async (prefilter gathers), MUFU = special-function unit, DFMA = fp64).  Run after esac_b200/build.py.
LIB=${1:-esac_b200/libesac_b200.so}
SASS=$(mktemp)
trap 'rm -f "$SASS"' EXIT
echo "cuobjdump -sass $LIB  ($(date -u +%Y-%m-%dT%H:%MZ), $(nvcc --version | tail -2 | head -1))"
echo "cubins: $(cuobjdump -lelf $LIB | grep -c sm_90a) x sm_90a"
cuobjdump -sass $LIB > "$SASS"
for m in UBLKCP SYNCS LDGSTS "LDGDEPBAR" FFMA FMUL FADD "MUFU.RSQ" "MUFU.EX2" "MUFU.RCP" "MUFU.RCP64H" "MUFU.RSQ64H" DFMA DMUL DADD "ATOM" "RED\." "SHFL" "BAR.SYNC" "LDG" "LDS" "STS" "ST.E.*STRONG.GPU" "LD.E.*STRONG.GPU" "MEMBAR"; do
  printf "%-22s %8d\n" "$m" "$(grep -cE "\b$m" "$SASS")"
done
echo
echo "per kernel (Function : name, then counts of UBLKCP / SYNCS / FFMA+FMUL+FADD / MUFU / DFMA):"
awk '/Function :/ {name=$3} /UBLKCP/ {u[name]++} /SYNCS/ {s[name]++} /FFMA|FMUL|FADD/ {f[name]++} /MUFU/ {m[name]++} /DFMA|DMUL|DADD/ {d[name]++} END {for (n in d) printf "%-110s UBLKCP %3d SYNCS %3d F32 %5d MUFU %4d FP64 %6d\n", substr(n,1,110), u[n], s[n], f[n], m[n], d[n]; for (n in f) if (!(n in d)) printf "%-110s UBLKCP %3d SYNCS %3d F32 %5d MUFU %4d FP64 %6d\n", substr(n,1,110), u[n], s[n], f[n], m[n], 0}' "$SASS" | sort
