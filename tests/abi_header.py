"""include/b200bt.h read for the ABI tests, and the refusal harness of the CPU-side entry-point tests.

parse() reads the C subset the header uses: integer #defines, enums, one pointer typedef, typedef structs of scalars and
arrays (dimensions may be macros), and prototypes.  A declaration outside that subset raises instead of being skipped,
so a new form in the header is noticed by the tests rather than left unchecked."""
import functools
import re
from pathlib import Path
from typing import NamedTuple, Optional, Tuple

HEADER_PATH = Path(__file__).resolve().parents[1] / "include" / "b200bt.h"
SCALARS = {"int": 4, "int32_t": 4, "uint32_t": 4, "float": 4, "double": 8, "int64_t": 8, "uint64_t": 8, "uint8_t": 1,
           "unsigned char": 1, "char": 1}


class CType(NamedTuple):
    base: str                    # a scalar, a struct or "void"; typedefs resolved
    pointers: int = 0


class Field(NamedTuple):
    name: str
    ctype: str                   # a scalar
    dims: Tuple[int, ...]
    offset: int
    size: int


class Struct(NamedTuple):
    fields: Tuple[Field, ...]
    size: int                    # natural alignment, as the C compiler lays it out
    comment: Optional[int]       # the "/* N bytes */" after the declaration


class Header(NamedTuple):
    prototypes: dict             # name -> (return CType, (parameter CType, ...))
    structs: dict                # typedef name -> Struct
    defines: dict                # macro or enumerator -> int


def _int_expr(text: str, defines: dict) -> int:
    expr = re.sub(r"\b(0[xX][0-9a-fA-F]+|\d+)[uUlL]*\b", lambda m: str(int(m.group(1), 0)), text)
    expr = re.sub(r"\bB200BT_\w+\b", lambda m: str(defines[m.group(0)]), expr)
    if not re.fullmatch(r"[\d\s()<>|&+\-*~]+", expr):
        raise ValueError(f"b200bt.h: not an integer expression: {text!r}")
    return int(eval(expr, {"__builtins__": {}}))


def _ctype(text: str, aliases: dict, structs: dict) -> CType:
    m = re.fullmatch(r"(?:const )?(\w+(?: \w+)?) ?(\**)", text.strip())
    if m is None:
        raise ValueError(f"b200bt.h: cannot parse the type {text!r}")
    base, pointers = m.group(1), len(m.group(2))
    if base in aliases:
        return CType(aliases[base].base, aliases[base].pointers + pointers)
    if base not in SCALARS and base not in structs and not (base == "void" and pointers):
        raise ValueError(f"b200bt.h: unknown type {text!r}")
    return CType(base, pointers)


def _struct(body: str, defines: dict, comment: Optional[int]) -> Struct:
    fields, offset, align = [], 0, 1
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        m = re.fullmatch(r"(unsigned char|\w+) (.+)", decl)
        if m is None or m.group(1) not in SCALARS:
            raise ValueError(f"b200bt.h: cannot parse the field {decl!r}")
        ctype, size = m.group(1), SCALARS[m.group(1)]
        for declarator in m.group(2).split(","):
            d = re.fullmatch(r"(\w+)((?: ?\[[^\]]+\])*)", declarator.strip())
            if d is None:
                raise ValueError(f"b200bt.h: cannot parse the field {declarator!r} of {decl!r}")
            dims = tuple(_int_expr(x, defines) for x in re.findall(r"\[([^\]]+)\]", d.group(2)))
            n = 1
            for x in dims:
                n *= x
            offset = -(-offset // size) * size
            fields.append(Field(d.group(1), ctype, dims, offset, size * n))
            offset += size * n
            align = max(align, size)
    return Struct(tuple(fields), -(-offset // align) * align, comment)


def _declarations(code: str):
    """The top-level declarations (up to a ';' outside braces), whitespace collapsed."""
    depth, start = 0, 0
    for i, ch in enumerate(code):
        depth += (ch == "{") - (ch == "}")
        if ch == ";" and depth == 0:
            yield " ".join(code[start:i].split())
            start = i + 1
    if code[start:].strip():
        raise ValueError(f"b200bt.h: unterminated declaration {code[start:].strip()[:80]!r}")


def _param(text: str, aliases: dict, structs: dict) -> CType:
    m = re.fullmatch(r"(.+?)\b\w+", text.strip())
    if m is None:
        raise ValueError(f"b200bt.h: cannot parse the parameter {text!r}")
    return _ctype(m.group(1), aliases, structs)


@functools.lru_cache(maxsize=None)
def parse(path: Path = HEADER_PATH) -> Header:
    raw = path.read_text()
    comments = {name: int(n) for name, n in re.findall(r"\}\s*(\w+)\s*;\s*/\*\s*(\d+) bytes\s*\*/", raw)}
    text = re.sub(r"/\*.*?\*/", lambda m: "\n" * m.group(0).count("\n") + " ", raw, flags=re.S)
    text = re.sub(r'#ifdef __cplusplus\s*(?:extern "C" \{|\})\s*#endif', "", text)
    defines, aliases, structs, prototypes = {}, {}, {}, {}
    code = []
    for line in text.splitlines():
        m = re.match(r"\s*#\s*(\w+)\s*(.*?)\s*$", line)
        if m is None:
            code.append(line)
        elif m.group(1) == "define":
            name, *value = m.group(2).split(None, 1)
            if value:                                                 # B200BT_H_, the include guard, has no value
                defines[name] = _int_expr(value[0], defines)
        elif m.group(1) not in ("ifndef", "endif", "include"):
            raise ValueError(f"b200bt.h: unexpected directive {line.strip()!r}")
    for decl in _declarations("\n".join(code)):
        if m := re.fullmatch(r"typedef struct (\w+) \{(.*)\} (\w+)", decl):
            if m.group(1) != m.group(3):
                raise ValueError(f"b200bt.h: struct tag {m.group(1)} differs from its typedef {m.group(3)}")
            structs[m.group(1)] = _struct(m.group(2), defines, comments.get(m.group(1)))
        elif m := re.fullmatch(r"typedef (.+?) ?(\w+)", decl):
            aliases[m.group(2)] = _ctype(m.group(1), aliases, structs)
        elif m := re.fullmatch(r"enum \w+ \{(.*)\}", decl):
            value = 0
            for item in filter(None, (x.strip() for x in m.group(1).split(","))):
                name, _, expr = (x.strip() for x in item.partition("="))
                value = _int_expr(expr, defines) if expr else value
                defines[name] = value
                value += 1
        elif m := re.fullmatch(r"(.+?) ?\b(b200bt_\w+) ?\((.*)\)", decl):
            params = () if m.group(3).strip() == "void" else tuple(
                _param(p, aliases, structs) for p in m.group(3).split(","))
            prototypes[m.group(2)] = (_ctype(m.group(1), aliases, structs), params)
        else:
            raise ValueError(f"b200bt.h: cannot parse the declaration {decl[:80]!r}")
    return Header(prototypes, structs, defines)


# -- refusal harness: the entry points check their arguments before the device, so a call with dummy pointers returns
# the refusal's status without a GPU (and without touching memory).

EINVAL, ENODEVICE, ELIMIT = (parse().defines[f"B200BT_{e}"] for e in ("EINVAL", "ENODEVICE", "ELIMIT"))
DEV = 1 << 20                    # a non-null, 16-byte aligned dummy device pointer that is never dereferenced


def status(name, *args):
    """Status of the C-ABI call `name(*args)`: 0 on success, else the code of its B200btError."""
    from ai_crypto_trader_b200 import _lib
    try:
        _lib.call(name, *args)
    except _lib.B200btError as e:
        return e.status
    return 0
