#!/usr/bin/env python3
"""Extract the string-form fixtures of the reference's wasm demo (wasm/index.js:2-8: inputs, CircuitString, the
Pinocchio SetupString in the older top-level-G1T layout, px strings) into tests/golden/wasm_index_strings.json.
Needs a checkout of the reference (located as in oracle/ref_binary.py); the tests read only the committed JSON."""
import json
import os
import re

import ref_binary

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "wasm_index_strings.json")


def const(src, name):
    m = re.search(r"^const %s = (.*?);?$" % name, src, re.M)
    return json.loads(re.sub(r"(\w+):", r'"\1":', m.group(1)) if name == "inputs" else m.group(1))


def main():
    src = open(os.path.join(ref_binary.require_reference_dir(), "wasm", "index.js")).read()
    i = src.index("const inputs = ")
    inputs_txt = src[i + len("const inputs = "):src.index("};", i) + 1]
    inputs = json.loads(re.sub(r"(\w+):", r'"\1":', inputs_txt))
    out = {"source": "wasm/index.js:2-8", "inputs": inputs, "circuit": const(src, "circuit"), "setup": const(src, "setup"),
           "px": const(src, "px")}
    json.dump(out, open(OUT, "w"))
    print("wrote", OUT, {k: (len(v) if hasattr(v, "__len__") else v) for k, v in out.items()})


if __name__ == "__main__":
    main()
