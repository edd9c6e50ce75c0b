#!/usr/bin/env python
"""Re-types the reference's render-test scene catalogue as Python (tests/golden/ref_scenes.py).

Reads integration-tests/src/render_tests/{simple,view,rescaler,tiles,transition,tiles_transitions}.rs of the
reference checkout given on the command line and translates the small Rust subset those files use -- struct literals with
`..Default::default()`, enum variants, vec!, Some/None, closures, helper functions, format! -- into Python source
that builds the same scenes through tests/ref_scene_rt.py.  The output is committed; tests never read the reference.

  python tools/retype_scenes.py REFERENCE_CHECKOUT > tests/golden/ref_scenes.py
"""
import os
import re
import sys

FILES = ["simple", "view", "rescaler", "tiles", "transition", "tiles_transitions"]

TOKEN = re.compile(r"""
    (?P<ws>\s+|//[^\n]*|/\*.*?\*/)
  | (?P<str>"(?:\\.|[^"\\])*")
  | (?P<num>0x[0-9a-fA-F_]+|\d[\d_]*\.\d[\d_]*(?:f32|f64)?|\d[\d_]*(?:\.(?![.\w]))?(?:usize|u32|u64|i32|f32|f64|u8)?)
  | (?P<id>[A-Za-z_][A-Za-z0-9_]*)
  | (?P<op>::|\.\.=|\.\.|=>|->|==|!=|<=|>=|&&|\|\||[{}()\[\],;:.|!?&=<>+\-*/#'])
""", re.X | re.S)


def tokenize(src):
    out, i = [], 0
    while i < len(src):
        m = TOKEN.match(src, i)
        if not m:
            raise SyntaxError(f"cannot tokenize at {src[i:i + 40]!r}")
        i = m.end()
        if m.lastgroup != "ws":
            out.append((m.lastgroup, m.group(m.lastgroup)))
    return out


class P:
    def __init__(self, toks):
        self.t, self.i = toks, 0
        self.hoisted = []

    def peek(self, k=0):
        return self.t[self.i + k] if self.i + k < len(self.t) else ("eof", "")

    def next(self):
        tok = self.peek()
        self.i += 1
        return tok

    def accept(self, v):
        if self.peek()[1] == v:
            self.i += 1
            return True
        return False

    def expect(self, v):
        if not self.accept(v):
            raise SyntaxError(f"expected {v!r}, got {self.peek()} near {' '.join(x[1] for x in self.t[max(0, self.i - 8):self.i + 4])}")

    # ---- types (skipped) ------------------------------------------------------------------------------------------
    def skip_type(self):
        depth = 0
        while True:
            k, v = self.peek()
            if v in ("<", "(", "["):
                depth += 1
            elif v in (">", ")", "]"):
                if depth == 0:
                    return
                depth -= 1
            elif depth == 0 and v in (",", "=", "{", ";", "|"):
                return
            elif k == "eof":
                return
            self.i += 1

    # ---- expressions ---------------------------------------------------------------------------------------------
    def expr(self):
        return self.binary(0)

    PREC = [("||",), ("&&",), ("==", "!=", "<", ">", "<=", ">="), ("..", "..="), ("+", "-"), ("*", "/")]

    def binary(self, level):
        if level == len(self.PREC):
            return self.unary()
        left = self.binary(level + 1)
        while self.peek()[1] in self.PREC[level]:
            op = self.next()[1]
            right = self.binary(level + 1)
            if op == "..":
                left = f"range({left}, {right})"
            elif op == "..=":
                left = f"range({left}, ({right}) + 1)"
            else:
                op = {"||": "or", "&&": "and"}.get(op, op)
                left = f"({left} {op} {right})"
        return left

    def unary(self):
        if self.accept("&"):
            self.accept("mut")
            return self.unary()
        if self.accept("-"):
            return f"(-{self.unary()})"
        if self.accept("!"):
            return f"(not {self.unary()})"
        return self.postfix(self.primary())

    def args(self, close):
        out = []
        while not self.accept(close):
            out.append(self.expr())
            if not self.accept(","):
                self.expect(close)
                break
        return out

    def postfix(self, e):
        while True:
            if self.accept("?"):
                continue
            if self.peek()[1] == "." and self.peek(1)[0] == "id":
                self.next()
                name = self.next()[1]
                if self.accept("("):
                    a = self.args(")")
                    if name in ("into", "clone", "to_string", "to_owned", "iter", "into_iter", "as_ref", "unwrap"):
                        pass
                    elif name == "collect":
                        e = f"list({e})"
                    elif name == "then":
                        e = f"(({a[0]})() if {e} else None)"
                    elif name == "map":
                        e = f"rt.rmap({e}, {a[0]})"
                    elif name == "max":
                        e = f"max({e}, {a[0]})"
                    else:
                        e = f"{e}.{name}({', '.join(a)})"
                else:
                    e = f"{e}.{name}"
                continue
            if self.peek()[1] == "(" and False:
                pass
            return e

    def block(self):
        """`{ stmts; tail }` as an expression"""
        self.expect("{")
        stmts, tail = [], "None"
        while not self.accept("}"):
            if self.peek()[1] == "let":
                stmts.append(self.let())
                continue
            e = self.expr()
            if self.accept(";"):
                stmts.append(("expr", e))
            else:
                self.expect("}")
                tail = e
                break
        if not stmts:
            return tail
        # hoist into a local function so that lets work
        name = f"_blk{len(self.hoisted)}"
        body = []
        for st in stmts:
            body.append(f"{st[1]} = {st[2]}" if st[0] == "let" else st[1])
        body.append(f"return {tail}")
        self.hoisted.append((name, body))
        return f"{name}()"

    def let(self):
        self.expect("let")
        self.accept("mut")
        name = self.next()[1]
        if self.accept(":"):
            self.skip_type()
        self.expect("=")
        e = self.expr()
        self.expect(";")
        return ("let", name, e)

    def closure(self):
        params = []
        while not self.accept("|"):
            self.accept("mut")
            params.append(self.next()[1])
            if self.accept(":"):
                self.skip_type()
            self.accept(",")
        if self.peek()[1] == "{":
            save = self.hoisted
            self.hoisted = []
            body = self.block()
            inner, self.hoisted = self.hoisted, save
            if inner:   # block with lets inside a closure: emit a def
                name = f"_clo{len(self.hoisted)}"
                lines = []
                for hn, hb in inner:
                    lines.append(f"def {hn}():")
                    lines += ["    " + x for x in hb]
                lines.append(f"return {body}")
                self.hoisted.append((name + "(" + ", ".join(params) + ")", lines))
                return name
            return f"(lambda {', '.join(params)}: {body})"
        return f"(lambda {', '.join(params)}: {self.expr()})"

    def primary(self):
        k, v = self.peek()
        if v == "|":
            self.next()
            return self.closure()
        if v == "||":
            self.next()
            if self.peek()[1] == "{":
                return f"(lambda: {self.block()})"
            return f"(lambda: {self.expr()})"
        if v == "(":
            self.next()
            items = self.args(")")
            return f"({items[0]})" if len(items) == 1 else "(" + ", ".join(items) + ("," if len(items) == 1 else "") + ")"
        if v == "{":
            return self.block()
        if v == "[":
            self.next()
            return "[" + ", ".join(self.args("]")) + "]"
        if v == "if":
            self.next()
            c = self.expr_no_struct()
            a = self.block()
            b = "None"
            if self.accept("else"):
                b = self.block() if self.peek()[1] == "{" else self.primary()
            return f"({a} if {c} else {b})"
        if k == "str":
            self.next()
            return v
        if k == "num":
            self.next()
            v = re.sub(r"(usize|u32|u64|i32|f32|f64|u8)$", "", v).replace("_", "")
            return v[:-1] + ".0" if v.endswith(".") else v
        if k == "id":
            return self.path()
        raise SyntaxError(f"unexpected token {self.peek()} near {' '.join(x[1] for x in self.t[max(0, self.i - 8):self.i + 4])}")

    no_struct = False

    def expr_no_struct(self):
        old, self.no_struct = self.no_struct, True
        e = self.expr()
        self.no_struct = old
        return e

    def path(self):
        parts = [self.next()[1]]
        while self.peek()[1] == "::":
            self.next()
            if self.peek()[1] == "<":   # turbofish
                self.next()
                self.skip_type()
                self.expect(">")
                continue
            parts.append(self.next()[1])
        name = ".".join(parts)
        if name in ("true", "false"):
            return name.capitalize()
        if name == "None":
            return "None"
        if self.peek()[1] == "!":   # macro
            self.next()
            close = {"[": "]", "(": ")", "{": "}"}[self.next()[1]]
            if parts[-1] == "vec":
                if self.accept(close):
                    return "[]"
                first = self.expr()
                if self.accept(";"):   # vec![x; n]
                    n = self.expr()
                    self.expect(close)
                    return f"[{first} for _ in range({n})]"
                items = [first]
                if self.accept(","):
                    items += self.args(close)
                else:
                    self.expect(close)
                return "[" + ", ".join(items) + "]"
            if parts[-1] == "format":
                a = self.args(close)
                fmt = a[0]
                if len(a) == 1:
                    return "f" + fmt
                return f"{fmt}.format({', '.join(a[1:])})"
            raise SyntaxError(f"macro {name}")
        if self.peek()[1] == "(":
            self.next()
            a = self.args(")")
            if name == "Some":
                return a[0]
            if name in ("Box.new", "Arc.new"):
                return a[0]
            return f"rt.{name}({', '.join(a)})" if parts[0][0].isupper() else f"{name}({', '.join(a)})"
        if self.peek()[1] == "{" and parts[-1][0].isupper() and not self.no_struct:
            self.next()
            fields = []
            while not self.accept("}"):
                if self.accept(".."):
                    self.expr()   # Default::default()
                    self.accept(",")
                    continue
                fname = self.next()[1]
                if self.accept(":"):
                    fields.append(f"{fname}={self.expr()}")
                else:
                    fields.append(f"{fname}={fname}")
                self.accept(",")
            return f"rt.{name}({', '.join(fields)})"
        if parts[0][0].isupper() and (len(parts) > 1 or not parts[0].isupper()):
            return f"rt.{name}"     # enum variant / associated constant
        return name                  # local, constant or function name

    # ---- items -----------------------------------------------------------------------------------------------------
    def items(self):
        out = []
        while self.peek()[0] != "eof":
            k, v = self.peek()
            if v == "#":   # attribute
                self.next()
                self.expect("[")
                depth = 1
                attr = []
                while depth:
                    t = self.next()[1]
                    depth += t == "["
                    depth -= t == "]"
                    attr.append(t)
                out.append(("attr", "".join(attr)))
                continue
            if v == "use" or v == "mod":
                while self.next()[1] != ";":
                    pass
                continue
            if v == "pub":
                self.next()
                if self.accept("("):
                    while self.next()[1] != ")":
                        pass
                continue
            if v == "const" or v == "static":
                self.next()
                name = self.next()[1]
                self.expect(":")
                self.skip_type()
                self.expect("=")
                e = self.expr()
                self.expect(";")
                out.append(("const", name, e))
                continue
            if v == "fn":
                self.next()
                name = self.next()[1]
                self.expect("(")
                params = []
                while not self.accept(")"):
                    self.accept("mut")
                    params.append(self.next()[1])
                    self.expect(":")
                    self.skip_type()
                    self.accept(",")
                if self.accept("->"):
                    self.skip_type()
                self.hoisted = []
                self.expect("{")
                body = []
                while not self.accept("}"):
                    if self.peek()[1] == "let":
                        st = self.let()
                        body += self.flush()
                        body.append(f"{st[1]} = {st[2]}")
                        continue
                    e = self.expr()
                    body += self.flush()
                    if self.accept(";"):
                        body.append(e)
                    else:
                        self.expect("}")
                        body.append(f"return {e}")
                        break
                out.append(("fn", name, params, body))
                continue
            raise SyntaxError(f"item {self.peek()}")
        return out

    def flush(self):
        lines = []
        for name, body in self.hoisted:
            lines.append(f"def {name if '(' in name else name + '()'}:")
            lines += ["    " + x for x in body]
        self.hoisted = []
        return lines


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: retype_scenes.py REFERENCE_CHECKOUT > tests/golden/ref_scenes.py")
    ref = sys.argv[1]
    base = os.path.join(ref, "integration-tests", "src", "render_tests")
    print('"""GENERATED by tools/retype_scenes.py from the reference\'s render tests (integration-tests/src/render_tests/')
    print('{' + ",".join(FILES) + '}.rs): the scene catalogue re-typed as Python.  Do not edit by hand."""')
    print("from tests import ref_scene_rt as rt")
    print()
    print("MODULES = {}")
    for mod in FILES:
        src = open(os.path.join(base, mod + ".rs")).read()
        items = P(tokenize(src)).items()
        print(f"\n\n# {'=' * 100}\n# {mod}.rs\n# {'=' * 100}")
        print(f"def _module_{mod}():")
        print("    MODULE, TESTS_ = " + repr(mod) + ", {}")
        print("    DEFAULT_RESOLUTION = rt.DEFAULT_RESOLUTION")
        is_test = False
        for it in items:
            if it[0] == "attr":
                is_test = it[1].startswith("render_test")
                continue
            if it[0] == "const":
                if it[1] == "TESTS":
                    continue
                print(f"    {it[1]} = {it[2]}")
            elif it[0] == "fn":
                _, name, params, body = it
                if is_test:
                    print(f"\n    def {name}(TEST_NAME={name!r}):")
                else:
                    print(f"\n    def {name}({', '.join(params)}):")
                for line in body:
                    print("        " + line)
                if is_test:
                    print(f"    TESTS_[{name!r}] = {name}")
                is_test = False
        print("    return TESTS_")
        print(f"MODULES[{mod!r}] = _module_{mod}()")


if __name__ == "__main__":
    main()
