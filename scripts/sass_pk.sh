#!/bin/bash
# Dev tool: per-source-line SASS instruction histogram of pk_decode_kernel (static count ~ dynamic count per phase).
#   scripts/sass_pk.sh [line_lo line_hi]      (needs controlar_b200/lib/libcontrolar_b200.so built with -lineinfo)
set -e
cd "$(dirname "$0")/.."
mkdir -p build/sass && cd build/sass
rm -f car_api*.cubin
cuobjdump -xelf all ../../controlar_b200/lib/libcontrolar_b200.so > /dev/null
nvdisasm -g -c car_api.sm_90a.cubin > _all.sass
a=$(grep -n "^\.text\._Z16pk_decode_kernel8PkParams:" _all.sass | cut -d: -f1)
b=$(awk -v a="$a" 'NR>a && /^\t\.section\t\.text\./ {print NR; exit}' _all.sass)
sed -n "${a},${b:-\$}p" _all.sass > pk.sass
python ../../scripts/sasshist.py pk.sass decode_persistent.cuh "${1:-0}" "${2:-100000}"
