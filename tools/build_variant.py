#!/usr/bin/env python
"""Build a tuning variant of libb200bt.so: tools/build_variant.py NAME -DFOO=1 ...  ->  gpurun_variants/NAME.so
(select it at run time with B200BT_LIB=<path>)."""
import subprocess, sys
from pathlib import Path
ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import __graft_entry__ as ge
name, flags = sys.argv[1], sys.argv[2:]
out = ROOT / "gpurun_variants"; out.mkdir(exist_ok=True)
bd = out / ("build_" + name); bd.mkdir(exist_ok=True)
procs, objs = [], []
for src in sorted(ge.CSRC.glob("*.cu")):
    obj = bd / (src.stem + ".o"); objs.append(obj)
    procs.append(subprocess.Popen([ge._nvcc(), *ge.NVCC_FLAGS, *flags, "-c", str(src), "-o", str(obj)]))
assert all(p.wait() == 0 for p in procs)
subprocess.check_call([ge._nvcc(), "-shared", *ge.ARCH, *map(str, objs), "-o", str(out / (name + ".so"))])
for o in objs: o.unlink()
bd.rmdir()
print(out / (name + ".so"))
