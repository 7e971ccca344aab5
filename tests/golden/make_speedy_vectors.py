"""Extracts the little-endian golden vectors of persia-speedy's own test suite
(rust/persia-speedy/tests/serialization_tests.rs of a PERSIA checkout, `symmetric_tests!` blocks) into
tests/golden/speedy_vectors.json, which the tests read:

    python tests/golden/make_speedy_vectors.py <path to the PERSIA checkout>

Only the literal byte lists are copied (test data, not code); the `in = ...` expressions are kept as text so that
tests/test_speedy_codec.py can show which Rust value each vector encodes."""
import json
import os
import re
import sys

SRC = "rust/persia-speedy/tests/serialization_tests.rs"
WANT = ["vec_u8", "vec_u16", "vec_u32", "vec_u64", "bool_false", "bool_true", "u16", "i16", "u32", "i32", "u64", "i64", "usize",
        "f32", "f64", "string", "tuple_u16_u16", "option_u16_some", "option_u16_none", "hashmap", "system_time", "derived_struct",
        "derived_simple_enum_a", "derived_simple_enum_b", "derived_simple_enum_c", "derived_enum_unit_variant",
        "derived_enum_tuple_variant", "derived_enum_struct_variant"]


def main():
    txt = open(os.path.join(sys.argv[1], SRC)).read()
    out = {}
    for name in WANT:
        m = re.search(r"\n\s*%s for ([^{]+?)\{\s*in = (.*?),\s*le = \[(.*?)\]" % re.escape(name), txt, re.S)
        assert m, name
        le = [int(x, 0) if not x.strip().startswith("0b") else int(x.strip().replace("_", ""), 0)
              for x in re.sub(r"//.*", "", m.group(3)).replace("\n", " ").split(",") if x.strip()]
        out[name] = {"type": " ".join(m.group(1).split()), "in": " ".join(m.group(2).split()), "le": le}
    dst = os.path.join(os.path.dirname(os.path.abspath(__file__)), "speedy_vectors.json")
    json.dump({"source": "rust/persia-speedy/tests/serialization_tests.rs (PersiaML/PERSIA @ ff754b8)", "vectors": out},
              open(dst, "w"), indent=1)
    print(dst, len(out))


if __name__ == "__main__":
    main()
