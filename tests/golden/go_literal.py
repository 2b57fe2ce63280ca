"""Minimal parser for Go composite literals, enough for the reference's table tests.

Used ONLY by tests/golden/gen_fixtures.py, which reads a checkout of the
reference to transcribe its Go test tables into JSON fixtures.  Nothing at
test run time imports this.

Grammar handled:
    value   := string | rawstring | number | '-' number | ident ('.' ident)* [call | literal]
             | '&' value | '[' ']' type literal | 'map' '[' type ']' type literal | literal | 'func' ...
    literal := '{' [ elem (',' elem)* [','] ] '}'
    elem    := [key ':'] value
Composite literals become {"__type": T, ...fields} (keyed) or lists (unkeyed);
identifiers become {"__ident": "pkg.Name"}; calls become {"__call": name, "args": [...]}.
"""
from __future__ import annotations

import re

_TOKEN = re.compile(
    r"""
    (?P<ws>\s+|//[^\n]*|/\*.*?\*/)
  | (?P<str>"(?:\\.|[^"\\])*")
  | (?P<raw>`[^`]*`)
  | (?P<num>(?:0x[0-9a-fA-F]+|\d+\.\d*(?:[eE][-+]?\d+)?|\.\d+|\d+(?:[eE][-+]?\d+)?))
  | (?P<id>[A-Za-z_][A-Za-z0-9_]*)
  | (?P<op>[{}\[\](),:.&*\-+/<>=!|%])
    """,
    re.X | re.S,
)


def tokenize(src: str):
    pos = 0
    out = []
    while pos < len(src):
        m = _TOKEN.match(src, pos)
        if not m:
            raise SyntaxError(f"bad char {src[pos]!r} at {pos}: {src[pos-30:pos+30]!r}")
        pos = m.end()
        k = m.lastgroup
        if k == "ws":
            continue
        out.append((k, m.group(k)))
    return out


class Parser:
    def __init__(self, toks, force_types=()):
        self.t = toks
        self.i = 0
        self.force_types = set(force_types)

    def peek(self, o=0):
        return self.t[self.i + o] if self.i + o < len(self.t) else ("eof", "")

    def eat(self, val=None):
        k, v = self.peek()
        if val is not None and v != val:
            raise SyntaxError(f"expected {val!r} got {v!r} at token {self.i}: {self.t[max(0,self.i-8):self.i+4]}")
        self.i += 1
        return k, v

    def parse_type(self) -> str:
        """Consume a type expression, return it as text."""
        parts = []
        while True:
            k, v = self.peek()
            if v == "[":
                self.eat()
                depth = 1
                s = "["
                while depth:
                    k2, v2 = self.eat()
                    if v2 == "[":
                        depth += 1
                    if v2 == "]":
                        depth -= 1
                    s += v2
                parts.append(s)
            elif v == "*":
                self.eat()
                parts.append("*")
            elif v == "map":
                self.eat()
                parts.append("map")
            elif k == "id":
                self.eat()
                name = v
                while self.peek()[1] == "." and self.peek(1)[0] == "id":
                    self.eat()
                    name += "." + self.eat()[1]
                parts.append(name)
                break
            else:
                break
        return "".join(parts)

    def parse_value(self):
        k, v = self.peek()
        if k == "str":
            self.eat()
            val = bytes(v[1:-1], "utf-8").decode("unicode_escape")
            return self._binop(val)
        if k == "raw":
            self.eat()
            return v[1:-1]
        if k == "num":
            self.eat()
            val = float(v) if any(c in v for c in ".eE") and not v.startswith("0x") else int(v, 0)
            return self._binop(val)
        if v == "-":
            self.eat()
            x = self.parse_value()
            return -x if isinstance(x, (int, float)) else {"__neg": x}
        if v == "&":
            self.eat()
            return self.parse_value()
        if v == "(":
            self.eat()
            inner = self.parse_value()
            self.eat(")")
            return self._binop(inner)
        if v == "{":
            return self.parse_literal(None)
        if v == "[" or v == "map" or v == "*":
            ty = self.parse_type()
            if self.peek()[1] == "{":
                return self.parse_literal(ty)
            if self.peek()[1] == "(":  # conversion like []string(x)
                return self.parse_call(ty)
            return {"__ident": ty}
        if v == "func":
            # skip function literal: func(...) ... { body }
            self.eat()
            depth = 0
            body = []
            while True:
                k2, v2 = self.eat()
                body.append(v2)
                if v2 == "{":
                    depth += 1
                elif v2 == "}":
                    depth -= 1
                    if depth == 0:
                        break
            if self.peek()[1] == "(":  # immediately invoked
                self.parse_call("func")
            return {"__func": " ".join(body)}
        if k == "id":
            self.eat()
            name = v
            while self.peek()[1] == "." and self.peek(1)[0] == "id":
                self.eat()
                name += "." + self.eat()[1]
            if self.peek()[1] == "{" and (self._looks_like_type(name) or name in self.force_types):
                return self.parse_literal(name)
            if self.peek()[1] == "(":
                return self._binop(self.parse_call(name))
            if self.peek()[1] == "[" and name in ("ptr.To", "pointer.To"):
                # generic instantiation ptr.To[int32](x)
                self.eat("[")
                self.parse_type()
                self.eat("]")
                return self.parse_call(name)
            if name == "true":
                return True
            if name == "false":
                return False
            if name == "nil":
                return None
            return self._binop({"__ident": name})
        raise SyntaxError(f"unexpected token {k} {v!r} at {self.i}: {self.t[max(0,self.i-8):self.i+4]}")

    def _binop(self, left):
        """Fold simple arithmetic on constants (e.g. 2 * 1000, time.Minute * 5)."""
        while self.peek()[1] in ("*", "+", "-", "/") and self.peek(1)[1] not in (",", "}", ")"):
            op = self.eat()[1]
            right = self.parse_value()
            if isinstance(left, (int, float)) and isinstance(right, (int, float)):
                left = {"*": left * right, "+": left + right, "-": left - right,
                        "/": left / right if right else 0}[op]
            else:
                left = {"__binop": op, "l": left, "r": right}
        return left

    @staticmethod
    def _looks_like_type(name: str) -> bool:
        last = name.split(".")[-1]
        return last[:1].isupper() or last in ("string", "int", "float64", "bool")

    def parse_call(self, name):
        self.eat("(")
        args = []
        while self.peek()[1] != ")":
            args.append(self.parse_value())
            if self.peek()[1] == ",":
                self.eat()
        self.eat(")")
        # pointer helpers: pointer.Int(2), ptr.To(3), pointer.Float64(...)
        low = name.lower()
        if (low.startswith("pointer.") or low.startswith("ptr.") or low.startswith("ptr_") or low in (
                "intptr", "int32ptr", "float64ptr")) and len(args) == 1:
            return args[0]
        if name in ("int", "int32", "int64", "float64", "uint64", "int32") and len(args) == 1:
            return args[0]
        return {"__call": name, "args": args}

    def parse_literal(self, ty):
        self.eat("{")
        keyed = {}
        items = []
        is_keyed = None
        while self.peek()[1] != "}":
            # try key ':' value
            save = self.i
            key = None
            try:
                k, v = self.peek()
                if k in ("id", "str") and self._find_colon_at_depth0():
                    if k == "id":
                        kk = self.parse_value()
                        key = kk["__ident"] if isinstance(kk, dict) and "__ident" in kk else str(kk)
                    else:
                        key = self.parse_value()
                    self.eat(":")
            except SyntaxError:
                self.i = save
                key = None
            val = self.parse_value()
            if key is not None:
                keyed[key] = val
                is_keyed = True
            else:
                items.append(val)
            if self.peek()[1] == ",":
                self.eat()
        self.eat("}")
        if is_keyed:
            if ty and not ty.startswith("map"):
                keyed["__type"] = ty
            return keyed
        return items

    def _find_colon_at_depth0(self) -> bool:
        """Is there a ':' before the next ',' or '}' at nesting depth 0 (from current token)?"""
        depth = 0
        j = self.i
        while j < len(self.t):
            v = self.t[j][1]
            if v in "{[(":
                depth += 1
            elif v in "}])":
                if depth == 0:
                    return False
                depth -= 1
            elif v == ":" and depth == 0:
                return True
            elif v == "," and depth == 0:
                return False
            j += 1
        return False


def find_literals(src: str, type_name: str):
    """Yield parsed literals for every `type_name{` occurrence in src (outermost only)."""
    out = []
    pos = 0
    pat = re.compile(re.escape(type_name) + r"\s*\{")
    while True:
        m = pat.search(src, pos)
        if not m:
            break
        start = m.start()
        # brace match on raw text (strings/comments aware) to find the end
        i = m.end() - 1
        depth = 0
        n = len(src)
        while i < n:
            c = src[i]
            if c == '"':
                i += 1
                while src[i] != '"':
                    i += 2 if src[i] == "\\" else 1
            elif c == "`":
                i = src.index("`", i + 1)
            elif src.startswith("//", i):
                i = src.index("\n", i)
            elif c == "{":
                depth += 1
            elif c == "}":
                depth -= 1
                if depth == 0:
                    break
            i += 1
        text = src[start:i + 1]
        toks = tokenize(text)
        p = Parser(toks, force_types=[type_name.split(']')[-1].lstrip('*')])
        out.append(p.parse_value())
        pos = i + 1
    return out
