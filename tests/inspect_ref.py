"""What `sylph-b200 inspect` should print, restated in Python from sylph's src/inspect.rs and the crates it serialises
with: serde_yaml 0.9.34 over unsafe-libyaml 0.2.11, floats by ryu 1.0.18 (versions of the reference's Cargo.lock).

The crate sources are not part of this repository, so the YAML rules below restate their documented behaviour
(parity unpinned beyond the reference's own `contains` checks):
* serde_yaml writes a string single-quoted when, read back plain, it would resolve to null, a bool, an integer
  (u128/i128, decimal or 0x/0o/0b), a float (Rust's f64 grammar, finite, or the YAML .inf/.nan spellings), or when it
  is "0" followed by digits; otherwise it asks libyaml for any style.
* libyaml writes a scalar plain unless its analysis forbids it (leading/trailing space, an indicator at the start,
  ": " or " #" inside, "---"/"..." at the start, line breaks, characters it does not print), then single-quoted unless
  that is forbidden too (unprintable characters, a space next to a break), then double-quoted with its escapes.
  The width is unlimited, so nothing is folded.  Strings with a line break are written double-quoted here (serde_yaml
  would use a literal block): see host/inspect.hpp.
* floats: ryu's shortest round-trip digits (numpy's Dragon4 in unique mode finds the same digits), laid out as plain
  decimal or d.ddde<exp> by ryu's thresholds for f32 and f64."""
import math
import os
import re
import struct

import numpy as np


class InvalidSketch(Exception):
    pass


# ---- reading (bincode 1.3: u64 lengths, 1-byte Option tags and bools, UTF-8 strings) ----

class _Buf:
    """a sketch file read front to back; k-mer arrays are skipped, not read"""

    def __init__(self, path):
        self.f = open(path, "rb")
        self.size = os.fstat(self.f.fileno()).st_size

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.f.close()

    def skip(self, n):
        if self.f.tell() + n > self.size:
            raise InvalidSketch("truncated")
        self.f.seek(n, os.SEEK_CUR)

    def take(self, n):
        v = self.f.read(n)
        if len(v) != n:
            raise InvalidSketch("truncated")
        return v

    def u64(self):
        return struct.unpack("<Q", self.take(8))[0]

    def flag(self):
        v = self.take(1)[0]
        if v > 1:
            raise InvalidSketch("bad tag")
        return v == 1

    def string(self):
        try:
            return self.take(self.u64()).decode("utf-8")
        except UnicodeDecodeError as e:
            raise InvalidSketch(str(e))


def read_database(path):
    """-> dict of DatabaseSketch (src/inspect.rs:69-76); the default one for a database without genomes"""
    genomes = []
    first = None
    with _Buf(path) as b:
        for _ in range(b.u64()):
            nk = b.u64()
            b.skip(8 * nk)
            if b.flag():
                b.skip(8 * b.u64())
            fn, contig = b.string(), b.string()
            c, k, gs, ms = b.u64(), b.u64(), b.u64(), b.u64()
            first = first or (c, k, ms)
            genomes.append(dict(file_name=fn, genome_kmers_num=nk, first_contig_name=contig, genome_size=gs))
    if not genomes:
        return dict(database_file="", c=0, k=0, min_spacing_parameter=0, genome_files=[])
    return dict(database_file=path, c=first[0], k=first[1], min_spacing_parameter=first[2], genome_files=genomes)


def read_sample(path):
    """-> dict of SequencesSketchInspect (src/inspect.rs:19-46)"""
    with _Buf(path) as b:
        n = b.u64()
        b.skip(12 * n)
        c, k = b.u64(), b.u64()
        fn = b.string()
        name = b.string() if b.flag() else None
        paired = b.flag()
        mrl = struct.unpack("<d", b.take(8))[0]
    f32 = np.float32
    with np.errstate(all="ignore"):
        anb = f32(mrl + float(k) - 1.) / f32(mrl) * f32(c) * f32(n)
    return dict(file_name=fn, c=c, k=k, num_sketched_kmers=n, approximate_number_bases=f32(anb), mean_read_length=mrl,
                sample_name=name, paired=paired)


# ---- serde_yaml: which strings would resolve to another scalar ----

_RADIX = re.compile(r"0x[0-9a-fA-F]+|0o[0-7]+|0b[01]+")
_FLOAT = re.compile(r"[+-]?([0-9]+\.?[0-9]*|\.[0-9]+)([eE][+-]?[0-9]+)?")


def _digits_but_not_number(s):
    t = s[1:] if s[:1] in ("+", "-") else s
    return len(t) > 1 and t[0] == "0" and t[1:].isascii() and t[1:].isdigit()


def _radix_value(t):
    return int(t[2:], {"x": 16, "o": 8, "b": 2}[t[1]])


def _is_int(s):
    u = s[1:] if s.startswith("+") else s
    if _RADIX.fullmatch(u) and _radix_value(u) < 2 ** 128:
        return True
    if not _digits_but_not_number(s) and re.fullmatch(r"[0-9]+", u) and int(u) < 2 ** 128:
        return True
    if s.startswith("-") and _RADIX.fullmatch(s[1:]) and _radix_value(s[1:]) <= 2 ** 127:
        return True
    if not _digits_but_not_number(s) and re.fullmatch(r"[+-]?[0-9]+", s):
        return -2 ** 127 <= int(s) < 2 ** 127
    return False


def _is_float(s):
    u = s
    if s.startswith("+"):
        u = s[1:]
        if u[:1] in ("+", "-"):
            return False
    if u in (".inf", ".Inf", ".INF") or s in ("-.inf", "-.Inf", "-.INF", ".nan", ".NaN", ".NAN"):
        return True
    return bool(_FLOAT.fullmatch(u)) and math.isfinite(float(u))


def resolves_to_other_scalar(s):
    return (s in ("", "~", "null", "Null", "NULL", "true", "True", "TRUE", "false", "False", "FALSE") or _is_int(s)
            or _digits_but_not_number(s) or _is_float(s))


# ---- libyaml: the scalar analysis and the quoted writers, on code points ----

_BREAKS = "\r\n\u0085\u2028\u2029"


def _printable(ch):
    cp = ord(ch)
    return cp == 0x0A or 0x20 <= cp <= 0x7E or 0xA0 <= cp <= 0xD7FF or (0xE000 <= cp <= 0xFFFD and cp != 0xFEFF)


def _blankz(s, i):
    return i >= len(s) or s[i] in " \t\0" or s[i] in _BREAKS


def _analysis(s):
    """-> (plain allowed in block context, single quotes allowed, has line breaks)"""
    if not s:
        return True, True, False
    indicator = s.startswith("---") or s.startswith("...")
    special = any(not _printable(ch) for ch in s)
    breaks = any(ch in _BREAKS for ch in s)
    for i, ch in enumerate(s):
        follows_ws = _blankz(s, i + 1)
        if i == 0:
            indicator |= ch in "#,[]{}&*!|>'\"%@`" or (ch in "?:-" and follows_ws)
        else:
            indicator |= (ch == ":" and follows_ws) or (ch == "#" and _blankz(s, i - 1))
    edge = s[0] == " " or s[-1] == " " or s[0] in _BREAKS or s[-1] in _BREAKS
    space_break = any(a == " " and b in _BREAKS for a, b in zip(s, s[1:]))
    break_space = any(a in _BREAKS and b == " " for a, b in zip(s, s[1:]))
    single = not (special or space_break or break_space)
    plain = single and not (edge or breaks or indicator)
    return plain, single, breaks


_ESC = {0x00: "0", 0x07: "a", 0x08: "b", 0x09: "t", 0x0A: "n", 0x0B: "v", 0x0C: "f", 0x0D: "r", 0x1B: "e", 0x22: '"',
        0x5C: "\\", 0x85: "N", 0xA0: "_", 0x2028: "L", 0x2029: "P"}


def _double_quoted(s):
    out = []
    for ch in s:
        cp = ord(ch)
        if not _printable(ch) or ch in _BREAKS or ch in '"\\':
            if cp in _ESC:
                out.append("\\" + _ESC[cp])
            elif cp <= 0xFF:
                out.append("\\x%02X" % cp)
            elif cp <= 0xFFFF:
                out.append("\\u%04X" % cp)
            else:
                out.append("\\U%08X" % cp)
        else:
            out.append(ch)
    return '"' + "".join(out) + '"'


def yaml_str(s):
    plain, single, breaks = _analysis(s)
    if breaks or not single:
        return _double_quoted(s)
    if plain and not resolves_to_other_scalar(s):
        return s
    return "'" + s.replace("'", "''") + "'"


def yaml_float(x, f32):
    """ryu's format32 / format64 of the shortest digits, after serde_yaml's .nan / .inf"""
    x = np.float32(x) if f32 else np.float64(x)
    if np.isnan(x):
        return ".nan"
    if np.isinf(x):
        return ".inf" if x > 0 else "-.inf"
    sign = "-" if np.signbit(x) else ""
    if x == 0:
        return sign + "0.0"
    mant, exp = np.format_float_scientific(abs(x), unique=True, trim="-").split("e")
    d = mant.replace(".", "")
    kk = int(exp) + 1                        # 10^(kk-1) <= |x| < 10^kk
    top, bottom = (13, -6) if f32 else (16, -5)
    if len(d) <= kk <= top:
        body = d + "0" * (kk - len(d)) + ".0"
    elif 0 < kk <= top:
        body = d[:kk] + "." + d[kk:]
    elif bottom < kk <= 0:
        body = "0." + "0" * -kk + d
    else:
        body = (d if len(d) == 1 else d[0] + "." + d[1:]) + "e%d" % (kk - 1)
    return sign + body


# ---- the documents ----

def databases_yaml(dbs):
    lines = []
    for d in dbs:
        lines += ["- database_file: " + yaml_str(d["database_file"]), "  c: %d" % d["c"], "  k: %d" % d["k"],
                  "  min_spacing_parameter: %d" % d["min_spacing_parameter"]]
        lines.append("  genome_files:" + ("" if d["genome_files"] else " []"))
        for g in d["genome_files"]:
            lines += ["  - file_name: " + yaml_str(g["file_name"]), "    genome_kmers_num: %d" % g["genome_kmers_num"],
                      "    first_contig_name: " + yaml_str(g["first_contig_name"]), "    genome_size: %d" % g["genome_size"]]
    return "".join(ln + "\n" for ln in lines)


def samples_yaml(samples):
    lines = []
    for s in samples:
        lines += ["- file_name: " + yaml_str(s["file_name"]), "  c: %d" % s["c"], "  k: %d" % s["k"],
                  "  num_sketched_kmers: %d" % s["num_sketched_kmers"],
                  "  approximate_number_bases: " + yaml_float(s["approximate_number_bases"], True),
                  "  mean_read_length: " + yaml_float(s["mean_read_length"], False),
                  "  sample_name: " + ("null" if s["sample_name"] is None else yaml_str(s["sample_name"])),
                  "  paired: " + ("true" if s["paired"] else "false")]
    return "".join(ln + "\n" for ln in lines)


def inspect(files):
    """the text `inspect files...` prints: every database (.syldb/.sylqueries), then every sample (.sylsp/.sylsample);
    other files are skipped"""
    dbs = [read_database(f) for f in files if f.endswith(".syldb") or f.endswith(".sylqueries")]
    samples = [read_sample(f) for f in files if f.endswith(".sylsp") or f.endswith(".sylsample")]
    return databases_yaml(dbs) + samples_yaml(samples)
