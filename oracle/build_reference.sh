#!/usr/bin/env bash
# Builds the unmodified reference CLI (b4rtaz/distributed-llama, `make dllama`) from a checkout given as $1 into oracle/_ref/dllama.
# The reference sources are copied to a temporary directory and built there; only the binary lands in oracle/_ref (git-ignored).
# Its Makefile uses -march=native: build on the machine that will run the binary (see oracle/README.md).
# Used by `bench.py --impl reference` and by oracle/make_golden.py, which regenerates tests/golden/reference_perplexity.json.
set -euo pipefail
SRC="${1:?usage: oracle/build_reference.sh <distributed-llama checkout>}"
OUT="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)/_ref"
WORK="$(mktemp -d)"
trap 'rm -rf "$WORK"' EXIT
cp -r "$SRC"/. "$WORK"/
make -C "$WORK" dllama -j"$(nproc)" > "$WORK/build.log" 2>&1 || { tail -30 "$WORK/build.log"; exit 1; }
mkdir -p "$OUT"
cp "$WORK/dllama" "$OUT/dllama"
echo "$OUT/dllama"
