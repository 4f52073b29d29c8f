#!/usr/bin/env python3
"""Transcribe the reference's golden search vectors into language-neutral JSON.

Run against a checkout of the reference crate (the tests only read the JSON written here):

    python tests/golden/extract_vectors.py <reference checkout> tests/golden

Sources (data only, no code is copied):
  * src/tests.rs:96-642        -> ac_vectors.json
  * src/packed/tests.rs:129-368 -> packed_vectors.json

Every `t!(name, &[patterns], "haystack", &[(pid, start, end), ...])` record in
a `const GROUP: &'static [SearchTest]` block becomes
  {"name":..., "patterns":[hex...], "haystack":hex, "matches":[[pid,s,e],...]}
with byte strings hex-encoded (the vectors contain NUL bytes).  Groups that the
reference keeps only inside a block comment (ANCHORED_OVERLAPPING) are skipped.
The collection tables (which groups run under which match semantics,
src/tests.rs:47-88 and src/packed/tests.rs:118-124) are recorded alongside.
"""
import json
import re
import sys
from pathlib import Path


def strip_block_comments(src: str) -> str:
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def parse_rust_str(s: str, i: int):
    """Parse a Rust "..." literal starting at s[i] == '"'. Returns (bytes, next_i)."""
    assert s[i] == '"'
    i += 1
    out = bytearray()
    while True:
        c = s[i]
        if c == '"':
            return bytes(out), i + 1
        if c == "\\":
            n = s[i + 1]
            if n == "x":
                out.append(int(s[i + 2:i + 4], 16))
                i += 4
            elif n == "n":
                out.append(10); i += 2
            elif n == "r":
                out.append(13); i += 2
            elif n == "t":
                out.append(9); i += 2
            elif n == "0":
                out.append(0); i += 2
            elif n in "\\\"'":
                out.append(ord(n)); i += 2
            else:
                raise ValueError(f"unsupported escape \\{n}")
        else:
            out += c.encode("utf-8")
            i += 1


def skip_ws(s, i):
    while s[i] in " \t\r\n":
        i += 1
    return i


def parse_group(body: str):
    tests = []
    i = 0
    while True:
        j = body.find("t!(", i)
        if j < 0:
            break
        i = j + 3
        i = skip_ws(body, i)
        m = re.match(r"[A-Za-z0-9_]+", body[i:])
        name = m.group(0)
        i += len(name)
        i = skip_ws(body, i); assert body[i] == ","; i += 1
        i = skip_ws(body, i); assert body[i:i + 2] == "&["; i += 2
        pats = []
        while True:
            i = skip_ws(body, i)
            if body[i] == "]":
                i += 1
                break
            if body[i] == ",":
                i += 1
                continue
            p, i = parse_rust_str(body, i)
            pats.append(p)
        i = skip_ws(body, i); assert body[i] == ","; i += 1
        i = skip_ws(body, i)
        hay, i = parse_rust_str(body, i)
        i = skip_ws(body, i); assert body[i] == ","; i += 1
        i = skip_ws(body, i); assert body[i:i + 2] == "&["; i += 2
        k = body.index("]", i)
        triples = re.findall(r"\(\s*(\d+)\s*,\s*(\d+)\s*,\s*(\d+)\s*,?\s*\)", body[i:k])
        i = k + 1
        tests.append({
            "name": name,
            "patterns": [p.hex() for p in pats],
            "haystack": hay.hex(),
            "matches": [[int(a), int(b), int(c)] for a, b, c in triples],
        })
    return tests


def parse_file(path: Path):
    src = strip_block_comments(path.read_text())
    groups = {}
    for m in re.finditer(r"const ([A-Z_]+): &'static \[SearchTest\] = &\[", src):
        start = m.end()
        end = src.index("\n];", start)
        groups[m.group(1)] = parse_group(src[start:end])
    collections = {}
    for m in re.finditer(r"const ([A-Z_]+): TestCollection =\s*&\[(.*?)\];", src, flags=re.S):
        collections[m.group(1)] = re.findall(r"[A-Z_]+", m.group(2))
    return {"groups": groups, "collections": collections}


def main():
    if len(sys.argv) < 2:
        sys.exit("usage: extract_vectors.py <reference checkout> [out dir]")
    ref = Path(sys.argv[1])
    out = Path(sys.argv[2] if len(sys.argv) > 2 else Path(__file__).parent)
    for src, dst in [("src/tests.rs", "ac_vectors.json"),
                     ("src/packed/tests.rs", "packed_vectors.json")]:
        data = parse_file(ref / src)
        data["source"] = f"BurntSushi/aho-corasick 1.1.3 {src}"
        n = sum(len(v) for v in data["groups"].values())
        (out / dst).write_text(json.dumps(data, indent=1) + "\n")
        print(f"{dst}: {len(data['groups'])} groups, {n} tests, collections={list(data['collections'])}")


if __name__ == "__main__":
    main()
