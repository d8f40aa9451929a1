# A/B harness for the GPU box (one `gpurun -- 'bash tools/gpu_ab.sh <spec-file>'` call = many variants on the same box).
# The spec file holds one variant per line:   <name> [ENV=VALUE ...] [-- bench.py args]
# e.g.   p1        B2S_LZ4_PIPE=1
#        p4_serial B2S_LZ4_PIPE=4 B2S_OVERLAP=0
# Every variant runs `bench.py --no-e2e --no-cpu --steps 4 --warmup 3` (device-resident) unless args are given; results
# land in gpurun_out/ab_<name>.json and a one-line summary is printed.  This is how the round-2 tables in
# profiles/r2_compress_generations.md / r2_tma_tokens.md were produced (env switches: csrc/api.cu, b2s_init).
spec=${1:-/dev/stdin}
while read -r name rest; do
  [ -z "$name" ] && continue
  case "$name" in \#*) continue;; esac
  envs=(); args=(--no-e2e --no-cpu --steps 4 --warmup 3); seen=0
  for tok in $rest; do
    if [ "$tok" = "--" ]; then seen=1; args=(); continue; fi
    if [ $seen = 1 ]; then args+=("$tok"); else envs+=("$tok"); fi
  done
  env "${envs[@]}" timeout 900 python bench.py "${args[@]}" > gpurun_out/ab_$name.json 2> gpurun_out/ab_$name.err
  python - "$name" <<'PY'
import json, sys
name = sys.argv[1]
try:
    d = [json.loads(l) for l in open("gpurun_out/ab_%s.json" % name) if l.startswith("{")][0]
    e = d.get("e2e") or {}
    print("== %-18s value %.2f GB/s  %.1f ms/step  ratio %s  kernels %s  e2e %s" % (
        name, d["value"], d["ms_per_step"], d.get("compressed_ratio"), d.get("kernels"), e.get("value")))
    for mode in ("serial", "concurrent"):
        m = e.get(mode)
        if m:
            print("   %-10s %.2f GB/s  %.1f ms/step  write %.1f ms  read %.1f ms  write sums %s  read sums %s" % (
                mode, m["value"], m["ms_per_step"], m["write_ms"], m["read_ms"], m["write_sums_ms"], m["read_sums_ms"]))
except Exception as ex:  # noqa: BLE001
    print("== %-18s FAILED: %r" % (name, ex))
PY
  tail -2 gpurun_out/ab_$name.err
done < "$spec"
