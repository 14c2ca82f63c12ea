#!/bin/bash
# TEST INFRASTRUCTURE.  Builds oracle/_ref/libxllm_ref.so = the reference's own hash / index / routing code
# (see oracle/ref_shim/ref_shim.cc for the file list), compiled UNMODIFIED from the reference checkout (XLLM_REFERENCE_DIR) with g++ against
# the stand-in headers in oracle/ref_shim/stubs.  Without that checkout the script does nothing and the tests use
# the prebuilt .so.  Outputs go to oracle/_ref/ only (git-ignored, shipped alongside the build).  No reference source is
# copied into the repository: the one generated file (the get_load_metrics cut) is deleted after compiling.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF="${XLLM_REFERENCE_DIR:-/root/reference}/xllm_service"
OUT="$HERE/_ref"
[ -d "$REF" ] || { echo "build_ref: $REF not found (prebuilt oracle/_ref is used as is)"; exit 0; }
SITE="$(python -c 'import sysconfig; print(sysconfig.get_paths()["purelib"])')"
XXH_INC="$SITE/pyarrow/include"                          # arrow/vendored/xxhash/xxhash.h (v0.8.3)
JSON_INC="$SITE/include/cudnn_frontend/thirdparty"       # nlohmann/json.hpp
[ -f "$XXH_INC/arrow/vendored/xxhash/xxhash.h" ] || { echo "build_ref: vendored xxhash.h not found"; exit 1; }
[ -f "$JSON_INC/nlohmann/json.hpp" ] || { echo "build_ref: nlohmann/json.hpp not found"; exit 1; }
mkdir -p "$OUT/obj"
ROOT="$(dirname "$HERE")"
SEAMS_SRCS=("$ROOT/tests/cpp/reference_seams_main.cc" "$ROOT/xllm_service_b200/host" "$ROOT/include")
if [ -f "$OUT/libxllm_ref.so" ] && [ -f "$OUT/reference_seams_test" ] &&
   [ -z "$(find "$HERE/ref_shim" "$HERE/build_ref.sh" "${SEAMS_SRCS[@]}" -newer "$OUT/reference_seams_test" -print -quit)" ] &&
   [ -z "$(find "$HERE/ref_shim" "$HERE/build_ref.sh" -newer "$OUT/libxllm_ref.so" -print -quit)" ]; then
  exit 0
fi
CXXFLAGS="-O2 -std=c++17 -fPIC -w -fno-access-control -I$HERE/ref_shim/stubs -I$REF -I$XXH_INC -I$JSON_INC"
# InstanceMgr::get_load_metrics and its helper, cut by line range (instance_mgr.cpp needs brpc as a whole)
GEN="$OUT/obj/instance_mgr_cut.cc"
{
  echo '#include <algorithm>'
  echo '#include "scheduler/managers/instance_mgr.h"'
  echo 'namespace xllm_service {'
  echo 'namespace {'
  sed -n '63,66p' "$REF/scheduler/managers/instance_mgr.cpp"
  echo '}'
  sed -n '287,359p' "$REF/scheduler/managers/instance_mgr.cpp"
  echo '}'
} > "$GEN"
grep -q 'void InstanceMgr::get_load_metrics' "$GEN" || { echo "build_ref: instance_mgr.cpp line ranges moved"; exit 1; }
grep -q 'bool is_instance_schedulable' "$GEN" || { echo "build_ref: instance_mgr.cpp line ranges moved"; exit 1; }
SRCS=(
  "$REF/common/hash_util.cpp"
  "$REF/common/global_gflags.cpp"
  "$REF/common/threadpool.cpp"
  "$REF/common/utils.cpp"
  "$REF/scheduler/etcd_client/etcd_client.cpp"
  "$REF/scheduler/managers/global_kvcache_mgr.cpp"
  "$REF/scheduler/loadbalance_policy/cache_aware_routing.cpp"
  "$GEN"
  "$HERE/ref_shim/ref_shim.cc"
)
OBJS=()
for s in "${SRCS[@]}"; do
  o="$OUT/obj/$(basename "$s").o"
  g++ $CXXFLAGS -c "$s" -o "$o" &
  OBJS+=("$o")
done
wait
g++ -shared -o "$OUT/libxllm_ref.so" "${OBJS[@]}" -lpthread
echo "build_ref: built $OUT/libxllm_ref.so"
# The boundary test: the reference's tokenizer/fast_tokenizer.cpp (unmodified) + host/reference_adaptors.h compiled
# against the reference's real tokenizer.h / slice.h / types.h / loadbalance_policy.h, linked with the product
# library and with libxllm_ref.so (the reference's GlobalKVCacheMgr / CacheAwareRouting to compare against).
if [ -f "$ROOT/xllm_service_b200/libxllm_ingest.so" ]; then
  g++ $CXXFLAGS -I"$REF/tokenizer" -I"$ROOT/xllm_service_b200/host" -I"$ROOT/include" \
      "$ROOT/tests/cpp/reference_seams_main.cc" "$REF/tokenizer/fast_tokenizer.cpp" \
      -o "$OUT/reference_seams_test" \
      -L"$OUT" -lxllm_ref -L"$ROOT/xllm_service_b200" -lxllm_ingest -lpthread \
      -Wl,-rpath,'$ORIGIN' -Wl,-rpath,'$ORIGIN/../../xllm_service_b200' -Wl,--allow-shlib-undefined
  echo "build_ref: built $OUT/reference_seams_test"
else
  echo "build_ref: libxllm_ingest.so not built yet; skipping reference_seams_test (run make lib first)"
fi
rm -rf "$OUT/obj"
