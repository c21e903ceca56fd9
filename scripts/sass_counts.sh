#!/bin/bash
# SASS evidence per compilation unit of libn1b200.so: which Hopper instructions each cubin contains.
# HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / wait, UTMALDG / UTMASTG = TMA bulk tensor load / store (.MULTICAST),
# SYNCS = mbarrier, HMMA = mma.sync (sm_80-class).
cd "$(dirname "$0")/../internnav_b200/_build" || exit 1
printf "%-22s %8s %10s %8s %8s %10s %7s %6s\n" unit HGMMA WARPGROUP UTMALDG UTMASTG MULTICAST SYNCS HMMA
for o in *.o; do
  s=$(cuobjdump -sass "$o" 2>/dev/null)
  c() { echo "$s" | grep -c "$1"; }
  printf "%-22s %8d %10d %8d %8d %10d %7d %6d\n" "${o%.o}" "$(c HGMMA)" "$(c WARPGROUP)" "$(c UTMALDG)" \
    "$(c UTMASTG)" "$(c 'UTMALDG.*MULTICAST')" "$(c SYNCS)" "$(c 'HMMA\.')"
done
