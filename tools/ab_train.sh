#!/bin/bash
# A/B of merge-loop launch geometry on one GPU: µs per merge and phase split (tools/probe_train.py) for each setting.
#   usage: tools/ab_train.sh [corpus: zipf|readme] [vocab] [bytes]
cd "$(dirname "$0")/.."
C=${1:-zipf}; V=${2:-32000}; B=${3:-100e6}
for t in 1024 512 256; do
  echo "== YTTM_LOOP_THREADS=$t"
  YTTM_LOOP_THREADS=$t python tools/probe_train.py "$C" "$V" "$B" 2>/dev/null | tail -1 | cut -c1-700
done
echo "== YTTM_TRAIN_PINNED_H2D=8 (corpus through two pinned staging buffers filled by 8 host threads; compare front_ms.h2d)"
YTTM_TRAIN_PINNED_H2D=8 python tools/probe_train.py "$C" "$V" "$B" 2>/dev/null | tail -1 | cut -c1-700
for b in 74 111; do
  echo "== YTTM_LOOP_BLOCKS=$b"
  YTTM_LOOP_BLOCKS=$b python tools/probe_train.py "$C" "$V" "$B" 2>/dev/null | tail -1 | cut -c1-700
done
echo "== YTTM_PAIR_MAX_LOAD_PCT=75 / 35 (default 50: rebuild above load 1/2, accept at 1/4)"
YTTM_PAIR_MAX_LOAD_PCT=75 python tools/probe_train.py "$C" "$V" "$B" 2>/dev/null | tail -1 | cut -c1-700
YTTM_PAIR_MAX_LOAD_PCT=35 python tools/probe_train.py "$C" "$V" "$B" 2>/dev/null | tail -1 | cut -c1-700
echo "== YTTM_DBG=8 (per-block apply / drain timers)"
YTTM_DBG=8 python tools/probe_train.py "$C" "$V" "$B" 2>/dev/null | tail -1 | cut -c1-900
