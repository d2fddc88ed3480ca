#!/bin/bash
# SASS evidence that the hot kernels use the tensor cores: per kernel, the count of each tensor-core / memory mnemonic in
# the built library (wgmma appears as HGMMA).   bash profiles/sass_listing.sh
cuobjdump -sass brainmagick_b200/libbm_b200.so 2>/dev/null | awk '
/Function :/ {name=$3}
/UTCHMMA|UTCQMMA|UTMALDG|UTMASTG|UTMAREDG|UTMAPF|UTCBAR|LDTM|STTM|UTCCP|ELECT/ {
  for (i = 1; i <= NF; i++) if ($i ~ /^(UTCHMMA|UTCQMMA|UTMALDG|UTMASTG|UTMAREDG|UTMAPF|UTCBAR|LDTM|STTM|UTCCP|ELECT)/) { gsub(/;/, "", $i); c[name " " $i]++ }
}
END { for (k in c) print c[k], k }' | sort -k2 | c++filt 2>/dev/null | awk '{n=$1; $1=""; printf "%5d %s\n", n, $0}'
