# A/B of two builds of libdad3d.so on the same box: headline step + per-layer table (diagnostics; DAD3D_LIB_PATH selects the build)
for v in old new old new; do
  echo "== $v"
  DAD3D_LIB_PATH=$PWD/dad_3dheads_b200/libdad3d_$v.so timeout 300 python bench.py --no-strict --no-extras --no-cpu-baseline 2>/dev/null | python -c "
import sys, json
d = json.loads(sys.stdin.read().strip().splitlines()[-1])
print(d['value'], d['ms_per_step'], d['clocks']['sm_mhz'], d['roofline']['kernel_ms_per_step'])
"
done
for v in old new; do
  DAD3D_LIB_PATH=$PWD/dad_3dheads_b200/libdad3d_$v.so timeout 300 python tools/layer_table.py --precision fp16x2 --out gpurun_out/r02_layers_ab_$v.md > /dev/null 2>&1
done
python - <<'PY'
import re
def rows(f):
    d = {}
    for l in open(f):
        p = [x.strip() for x in l.split('|')]
        if len(p) > 10 and p[1] not in ('layer', '---'):
            try: d[p[1]] = float(p[9])
            except ValueError: pass
    return d
a, b = rows('gpurun_out/r02_layers_ab_old.md'), rows('gpurun_out/r02_layers_ab_new.md')
print('layer old_us new_us')
for k in a:
    if k in b and abs(a[k] - b[k]) > 0.03 * a[k]: print(k, a[k], b[k])
print('sum', sum(a.values()), sum(b.values()))
PY
