#!/bin/bash
# Pin the oracle against the REAL reference.  Needs cargo + crates.io access — run it on any machine with a
# Rust toolchain and commit the two JSON files it writes; tests/test_oracle_cpu.py::test_reference_goldens then
# compares the oracle with them (it skips while they are absent).
#   usage: tools/run_reference.sh /path/to/cozo            (the repository root that holds cozo-core/)
set -euo pipefail
REF="${1:?usage: tools/run_reference.sh /path/to/cozo}"
HERE="$(cd "$(dirname "$0")/.." && pwd)"
command -v cargo >/dev/null || { echo "cargo not found: this script needs a Rust toolchain" >&2; exit 2; }
TMP="$(mktemp -d)"
python "$HERE/tests/golden/make_reference_inputs.py" "$TMP"
sed "s#path = \"../../../reference/cozo-core\"#path = \"$REF/cozo-core\"#" "$HERE/tools/reference_golden/Cargo.toml" > "$TMP/Cargo.toml"
mkdir -p "$TMP/src" && cp "$HERE/tools/reference_golden/src/main.rs" "$TMP/src/"
(cd "$TMP" && cargo run --release -- "$TMP" "$REF/cozo-core/tests" "$HERE/tests/golden")
ls -la "$HERE/tests/golden/reference_hnsw.json" "$HERE/tests/golden/reference_graph.json"
