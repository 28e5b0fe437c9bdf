"""No float atomics in the CUDA sources: a float sum whose order depends on scheduling gives different bits from run to run
(integer atomics are exact in any order and stay allowed)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "hi3d_official_b200", "csrc")

ATOMIC_CALL = re.compile(r"\batomic(?:Add|Sub|Max|Min|Exch)(?:_block|_system)?\s*\(\s*&?\s*\(?\s*([A-Za-z_]\w*)")
# PTX reductions / atomics on floating-point types, e.g. red.global.add.f32, atom.shared.add.noftz.f16x2
PTX_FLOAT_ATOMIC = re.compile(r"\b(?:red|atom)(?:\.[a-z0-9_:]+)*\.(?:f16|f16x2|bf16|bf16x2|f32|f64)\b")
FLOAT_TYPES = r"(?:float|double|__half|__half2|half|half2|__nv_bfloat16|__nv_bfloat162|float2|float4)"


def float_atomics(src: str):
    """(line, text) of every float atomic in one CUDA source: atomic calls on a name declared with a floating-point type, and
    PTX red / atom instructions on floating-point types."""
    hits = []
    lines = src.splitlines()
    for m in ATOMIC_CALL.finditer(src):
        name = m.group(1)
        decl = re.compile(FLOAT_TYPES + r"\s*(?:\*\s*)?(?:const\s+)?(?:__restrict__\s+)?" + re.escape(name) + r"\s*[\[,;=)]")
        if decl.search(src):
            ln = src.count("\n", 0, m.start())
            hits.append((ln + 1, lines[ln].strip()))
    for m in PTX_FLOAT_ATOMIC.finditer(src):
        ln = src.count("\n", 0, m.start())
        hits.append((ln + 1, lines[ln].strip()))
    return hits


def test_scanner_finds_float_atomics():
    shared = "__shared__ float su[64];\n  atomicAdd(&su[2 * u], a);\n"
    table = "void k(float* __restrict__ stats) {\n  atomicAdd(&stats[i], v);\n}\n"
    ptx = 'asm volatile("red.global.add.f32 [%0], %1;" :: "l"(p), "f"(v));\n'
    integer = "__shared__ int cnt;\n  atomicAdd(&cnt, 1);\n  asm(\"red.global.add.u32 [%0], 1;\" :: \"l\"(p));\n"
    assert len(float_atomics(shared)) == 1 and len(float_atomics(table)) == 1 and len(float_atomics(ptx)) == 1
    assert float_atomics(integer) == []


def test_no_float_atomics_in_csrc():
    found = []
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            with open(os.path.join(CSRC, f)) as fh:
                found += [f"{f}:{ln}: {t}" for ln, t in float_atomics(fh.read())]
    assert not found, "float atomics make results depend on scheduling:\n" + "\n".join(found)
