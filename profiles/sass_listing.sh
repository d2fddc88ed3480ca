#!/bin/bash
# SASS evidence for the sm_90a build: per kernel, the count of each tensor-core / memory instruction of interest in the
# built library -- HGMMA (wgmma), ATOMS.CAST.SPIN* (a shared-memory atomic the hardware has no native form of, e.g. an fp64
# add: a compare-and-swap loop), STG.E* / LDG.E* by width, and REDG* (global reductions: atomics without a return value).
#   bash profiles/sass_listing.sh [library]        (default: brainmagick_b200/libbm_b200.so)
cuobjdump -sass "${1:-brainmagick_b200/libbm_b200.so}" 2>/dev/null | awk '
/Function :/ {name=$3; next}
/^ *\/\*[0-9a-f]+\*\// {
  i = 2
  if ($i ~ /^@/) i++                          # a predicate guard
  op = $i; gsub(/;/, "", op)
  if (op ~ /^HGMMA/) op = "HGMMA"
  if (op ~ /^(HGMMA|ATOMS\.CAST\.SPIN|STG\.E|LDG\.E|REDG)/) c[name " " op]++
}
END { for (k in c) print c[k], k }' | sort -k2 | c++filt 2>/dev/null | awk '{n=$1; $1=""; printf "%5d %s\n", n, $0}'
