// wgsl.cpp -- WGSL lexer, parser, type checker, header validation and CUDA C++ emitter (see wgsl.h).
//
// The emitted module is compiled after wgsl_rt.cuh, whose functions carry WGSL's integer, conversion and indexing rules.
// Abstract-int and abstract-float expressions are evaluated here (in int64 / double, as WGSL's const-expressions are) and
// emitted as literals of the concrete type their context gives them; a `let` or a call argument without such a context
// takes i32 / f32.  Names of the module are prefixed (u_ values, S_ structs, m_ members, fn_ functions) so that they
// cannot collide with C++ or with the runtime.
#include "wgsl.h"

#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <set>
#include <vector>

#include "../../include/smelter_b200.h"

namespace smr {
namespace wgsl {
namespace {

struct Fail {
    int status;
    std::string msg;
};
[[noreturn]] void fail(int status, int line, int col, const std::string &m) {
    throw Fail{status, std::to_string(line) + ":" + std::to_string(col) + ": " + m};
}
[[noreturn]] void invalid(int line, int col, const std::string &m) { fail(SMR_ERR_INVALID_ARGUMENT, line, col, m); }
[[noreturn]] void unsupported(int line, int col, const std::string &m) { fail(SMR_ERR_UNSUPPORTED, line, col, "unsupported: " + m); }

// ---------------------------------------------------------------------------------------------------------------- lexer
struct Tok {
    enum K { Id, Int, Float, Punct, End } k = End;
    std::string s;      // identifier / punctuation / literal suffix
    long long iv = 0;
    double fv = 0;
    int line = 1, col = 1;
};

// A hexadecimal float literal ("0x" digits ["." digits] ["p" exponent]) must be exactly representable: in f32 with the f
// suffix, in f64 (abstract-float) without it.  Anything else is refused, as hexf-style parsers without rounding do.
double hex_float(const std::string &num, bool f32, int line, int col) {
    unsigned long long m = 0;
    long long e2 = 0;
    int sig = 0;   // significant hex digits in m
    bool frac = false, inexact = false;
    size_t i = 2;
    for (; i < num.size() && num[i] != 'p' && num[i] != 'P'; i++) {
        if (num[i] == '.') { frac = true; continue; }
        const int d = isdigit((unsigned char)num[i]) ? num[i] - '0' : (tolower((unsigned char)num[i]) - 'a' + 10);
        if (sig < 16) {
            if (m || d) { m = m * 16 + d; sig++; }
            if (frac) e2 -= 4;
        } else {
            inexact = inexact || d;   // past 61 significant bits: more than any f64 holds
            if (!frac) e2 += 4;
        }
    }
    if (i < num.size()) {
        const long long e = strtoll(num.c_str() + i + 1, nullptr, 10);   // saturates; a huge exponent is out of range below
        e2 += std::max(-100000LL, std::min(100000LL, e));
    }
    const char *what = f32 ? "f32" : "abstract-float (f64)";
    if (inexact) invalid(line, col, std::string("hexadecimal float literal is not exactly representable in ") + what);
    if (!m) return 0.0;
    while (!(m & 1)) { m >>= 1; e2++; }
    int bits = 0;
    for (unsigned long long v = m; v; v >>= 1) bits++;
    const int p = f32 ? 24 : 53, emin = f32 ? -126 : -1022, emax = f32 ? 127 : 1023;
    const long long top = e2 + bits - 1;
    if (top > emax) invalid(line, col, std::string("hexadecimal float literal out of the range of ") + what);
    if (bits > p || e2 < emin - (p - 1)) invalid(line, col, std::string("hexadecimal float literal is not exactly representable in ") + what);
    return std::ldexp((double)m, (int)e2);
}

std::vector<Tok> lex(const std::string &src) {
    std::vector<Tok> out;
    size_t i = 0;
    int line = 1, col = 1;
    auto adv = [&](size_t n) {
        for (size_t k = 0; k < n && i < src.size(); k++, i++) {
            if (src[i] == '\n') { line++; col = 1; } else col++;
        }
    };
    static const char *puncts[] = {"<<=", ">>=", "->", "&&", "||", "==", "!=", "<=", ">=", "+=", "-=", "*=", "/=", "%=", "&=",
                                   "|=", "^=", "++", "--", "<<", ">>", "(", ")", "{", "}", "[", "]", "<", ">", ",", ";", ":",
                                   ".", "=", "+", "-", "*", "/", "%", "&", "|", "^", "~", "!", "@", "_"};
    while (i < src.size()) {
        char c = src[i];
        if (c == ' ' || c == '\t' || c == '\r' || c == '\n' || c == '\v' || c == '\f') { adv(1); continue; }
        if (c == '/' && i + 1 < src.size() && src[i + 1] == '/') {
            while (i < src.size() && src[i] != '\n') adv(1);
            continue;
        }
        if (c == '/' && i + 1 < src.size() && src[i + 1] == '*') {
            int l0 = line, c0 = col, depth = 0;
            do {
                if (i + 1 >= src.size()) invalid(l0, c0, "unterminated block comment");
                if (src[i] == '/' && src[i + 1] == '*') { depth++; adv(2); }
                else if (src[i] == '*' && src[i + 1] == '/') { depth--; adv(2); }
                else adv(1);
            } while (depth > 0);
            continue;
        }
        Tok t;
        t.line = line; t.col = col;
        if (isalpha((unsigned char)c) || (c == '_' && i + 1 < src.size() && (isalnum((unsigned char)src[i + 1]) || src[i + 1] == '_'))) {
            size_t j = i;
            while (j < src.size() && (isalnum((unsigned char)src[j]) || src[j] == '_')) j++;
            t.k = Tok::Id; t.s = src.substr(i, j - i);
            adv(j - i);
            out.push_back(t);
            continue;
        }
        if (isdigit((unsigned char)c) || (c == '.' && i + 1 < src.size() && isdigit((unsigned char)src[i + 1]))) {
            size_t j = i;
            bool hex = c == '0' && i + 1 < src.size() && (src[i + 1] == 'x' || src[i + 1] == 'X');
            bool isf = false;
            if (hex) {   // 0x1f is an integer; 0x1.8, 0x.8p0 and 0X1P-2f are floats (without an exponent, f is a digit)
                j += 2;
                size_t digits = 0;
                for (; j < src.size() && isxdigit((unsigned char)src[j]); j++) digits++;
                if (j < src.size() && src[j] == '.') {
                    isf = true;
                    for (j++; j < src.size() && isxdigit((unsigned char)src[j]); j++) digits++;
                }
                if (j < src.size() && (src[j] == 'p' || src[j] == 'P')) {
                    isf = true;
                    j++;
                    if (j < src.size() && (src[j] == '+' || src[j] == '-')) j++;
                    if (j >= src.size() || !isdigit((unsigned char)src[j])) invalid(line, col, "malformed number");
                    while (j < src.size() && isdigit((unsigned char)src[j])) j++;
                }
                if (!digits) invalid(line, col, "malformed number");
            } else {
                while (j < src.size() && isdigit((unsigned char)src[j])) j++;
                if (j < src.size() && src[j] == '.') { isf = true; j++; while (j < src.size() && isdigit((unsigned char)src[j])) j++; }
                if (j < src.size() && (src[j] == 'e' || src[j] == 'E')) {
                    size_t k = j + 1;
                    if (k < src.size() && (src[k] == '+' || src[k] == '-')) k++;
                    if (k < src.size() && isdigit((unsigned char)src[k])) {
                        isf = true;
                        j = k;
                        while (j < src.size() && isdigit((unsigned char)src[j])) j++;
                    }
                }
            }
            std::string num = src.substr(i, j - i);
            std::string suf;
            if (j < src.size() && (src[j] == 'i' || src[j] == 'u' || src[j] == 'f' || src[j] == 'h')) suf = src[j++];
            if (j < src.size() && (isalnum((unsigned char)src[j]) || src[j] == '_')) invalid(line, col, "malformed number");
            if (suf == "h") unsupported(line, col, "f16 literals");
            if (isf || suf == "f") {
                t.k = Tok::Float;
                if (hex && suf != "" && suf != "f") invalid(line, col, "malformed number");
                t.fv = hex ? hex_float(num, suf == "f", line, col) : strtod(num.c_str(), nullptr);
            } else {
                t.k = Tok::Int;
                errno = 0;
                unsigned long long v = strtoull(num.c_str(), nullptr, hex ? 16 : 10);
                if (errno || v > 0x7fffffffffffffffull) invalid(line, col, "integer literal out of range");
                if (!hex && num.size() > 1 && num[0] == '0') invalid(line, col, "integer literal with a leading zero");
                t.iv = (long long)v;
            }
            t.s = suf;
            adv(j - i);
            out.push_back(t);
            continue;
        }
        bool found = false;
        for (const char *p : puncts) {
            size_t n = strlen(p);
            if (src.compare(i, n, p) == 0) {
                t.k = Tok::Punct; t.s = p;
                adv(n);
                out.push_back(t);
                found = true;
                break;
            }
        }
        if (!found) invalid(line, col, std::string("unexpected character '") + c + "'");
    }
    Tok e;
    e.line = line; e.col = col;
    out.push_back(e);
    return out;
}

// ------------------------------------------------------------------------------------------------------------------ AST
struct Expr;
struct TypeExpr;
using ExprP = std::shared_ptr<Expr>;
using TypeP = std::shared_ptr<TypeExpr>;

struct TypeExpr {                 // a type as written: name<args>; an argument is a type or an expression (array size)
    std::string name;
    std::vector<TypeP> targs;
    std::vector<ExprP> eargs;     // parallel to targs: the expression when the argument is not a type
    int line = 0, col = 0;
};

struct Attr {
    std::string name;
    std::vector<std::string> args;   // identifiers and integers, as written
    int line = 0, col = 0;
};
using Attrs = std::vector<Attr>;
const Attr *find_attr(const Attrs &a, const char *n) {
    for (const Attr &x : a) if (x.name == n) return &x;
    return nullptr;
}

// scalar kinds; AI / AF are abstract-int and abstract-float
enum SK { S_BOOL, S_I32, S_U32, S_F32, S_AI, S_AF };
struct Ty {
    enum K { Void, Scalar, Vec, Mat, Arr, Struct, Tex, Samp, TexArr } k = Void;
    SK s = S_F32;   // Scalar, Vec, Mat: the element
    int n = 0;      // Vec: size; Mat: columns; Arr / TexArr: length
    int m = 0;      // Mat: rows
    std::shared_ptr<Ty> el;   // Arr
    int sid = -1;   // Struct
};
bool operator==(const Ty &a, const Ty &b) {
    if (a.k != b.k || a.n != b.n || a.m != b.m || a.sid != b.sid) return false;
    if ((a.k == Ty::Scalar || a.k == Ty::Vec || a.k == Ty::Mat) && a.s != b.s) return false;
    if (a.k == Ty::Arr) return *a.el == *b.el;
    return true;
}
bool operator!=(const Ty &a, const Ty &b) { return !(a == b); }
Ty scalar(SK s) { Ty t; t.k = Ty::Scalar; t.s = s; return t; }
Ty vec(SK s, int n) { Ty t; t.k = Ty::Vec; t.s = s; t.n = n; return t; }
Ty with_elem(const Ty &t, SK s) { Ty r = t; r.s = s; return r; }
bool abstract(const Ty &t) { return (t.k == Ty::Scalar || t.k == Ty::Vec) && (t.s == S_AI || t.s == S_AF); }
bool numeric(SK s) { return s != S_BOOL; }
bool integral(SK s) { return s == S_I32 || s == S_U32 || s == S_AI; }
SK concrete_of(SK s) { return s == S_AI ? S_I32 : s == S_AF ? S_F32 : s; }
Ty concrete(const Ty &t) { return abstract(t) ? with_elem(t, concrete_of(t.s)) : t; }

// an abstract value: a scalar (n = 0) or a vector
struct CV {
    bool f = false;
    int n = 0;
    double fv[4] = {0, 0, 0, 0};
    long long iv[4] = {0, 0, 0, 0};
};

struct Expr {
    enum K { Lit, Id, Un, Bin, Call, Idx, Mem } k = Lit;
    int line = 0, col = 0;
    std::string s;                // Id: name; Un / Bin: operator; Mem: member
    TypeP callee;                 // Call
    std::vector<ExprP> a;         // operands / arguments
    char lk = 0;                  // Lit: 'b' bool, 'i' int, 'f' float
    std::string suf;              // Lit: suffix
    long long iv = 0;
    double fv = 0;
    bool bv = false;
    // filled by the checker
    Ty ty;
    bool has_cv = false;
    CV cv;
    bool has_target = false;
    Ty target;
    std::string code;             // what emit() returns when not an abstract value
    bool uref = false;            // the uniform, or a member / element of it: `code` is its byte offset
    bool cint = false;            // a concrete integer constant (suffixed literal or const), whose value is civ
    long long civ = 0;
};

struct Stmt;
using StmtP = std::shared_ptr<Stmt>;
struct Clause {
    std::vector<ExprP> sels;
    bool def = false;
    std::vector<StmtP> body;
};
struct Stmt {
    enum K { Block, Var, Let, Const, Assign, Incr, Decr, If, Switch, Loop, For, While, Break, BreakIf, Continue, Return,
             Discard, CallS, Phony, ConstAssert } k = Block;
    int line = 0, col = 0;
    std::string name, op;
    TypeP ty;
    ExprP e, lhs;
    std::vector<StmtP> body, cont;   // Block / loop body; Loop: continuing
    StmtP els, init, update;         // If: else (Block or If); For: init, update
    std::vector<Clause> clauses;
};

struct Member {
    std::string name;
    TypeP ty;
    Attrs attrs;
    int line = 0, col = 0;
};
struct StructDecl {
    std::string name;
    std::vector<Member> members;
    int line = 0, col = 0;
};
struct Global {
    std::string name, space, access;
    TypeP ty;
    ExprP init;
    Attrs attrs;
    int line = 0, col = 0;
};
struct ConstDecl {
    std::string name;
    TypeP ty;
    ExprP init;
    int line = 0, col = 0;
};
struct Param {
    std::string name;
    TypeP ty;
    Attrs attrs;
    int line = 0, col = 0;
};
struct FnDecl {
    std::string name;
    std::vector<Param> params;
    TypeP ret;
    Attrs attrs, ret_attrs;
    std::vector<StmtP> body;
    int line = 0, col = 0;
};
struct AliasDecl {
    std::string name;
    TypeP ty;
    int line = 0, col = 0;
};
struct Module {
    std::vector<StructDecl> structs;
    std::vector<Global> globals;
    std::vector<ConstDecl> consts;
    std::vector<FnDecl> fns;
    std::vector<AliasDecl> aliases;
    std::vector<StmtP> asserts;   // module-scope const_assert
};

// ---------------------------------------------------------------------------------------------------------------- parser
const std::set<std::string> kTemplated = {"vec2", "vec3", "vec4", "mat2x2", "mat2x3", "mat2x4", "mat3x2", "mat3x3", "mat3x4",
                                          "mat4x2", "mat4x3", "mat4x4", "array", "bitcast", "ptr", "atomic", "binding_array",
                                          "texture_1d", "texture_2d", "texture_2d_array", "texture_3d", "texture_cube",
                                          "texture_cube_array", "texture_multisampled_2d", "texture_storage_1d",
                                          "texture_storage_2d", "texture_storage_2d_array", "texture_storage_3d"};

struct Parser {
    std::vector<Tok> t;
    size_t p = 0;
    Module m;

    const Tok &cur() const { return t[p]; }
    bool is(const char *s) const { return t[p].k == Tok::Punct && t[p].s == s; }
    bool is_id(const char *s) const { return t[p].k == Tok::Id && t[p].s == s; }
    [[noreturn]] void err(const std::string &m) const { invalid(cur().line, cur().col, m); }
    void expect(const char *s) {
        if (!is(s)) err(std::string("expected '") + s + "', found '" + (cur().k == Tok::End ? "end of file" : cur().s) + "'");
        p++;
    }
    bool accept(const char *s) {
        if (is(s)) { p++; return true; }
        return false;
    }
    std::string ident() {
        if (cur().k != Tok::Id) err("expected an identifier");
        return t[p++].s;
    }

    // diagnostic(severity, rule) of a directive or an attribute: {severity, rule}; the rule may be namespaced (a.b)
    std::vector<std::string> diagnostic_args() {
        expect("(");
        int line = cur().line, col = cur().col;
        std::string sev = ident();
        if (sev != "error" && sev != "warning" && sev != "info" && sev != "off")
            invalid(line, col, "unknown diagnostic severity '" + sev + "'");
        expect(",");
        std::string rule = ident();
        if (accept(".")) rule += "." + ident();
        accept(",");
        expect(")");
        return {sev, rule};
    }
    // diagnostic filters on one range conflict when they give one rule two severities
    std::map<std::string, std::string> module_diagnostics;
    static void diagnostic_filter(std::map<std::string, std::string> &seen, const std::vector<std::string> &d, int line, int col) {
        auto it = seen.find(d[1]);
        if (it != seen.end() && it->second != d[0]) invalid(line, col, "conflicting diagnostic filters for '" + d[1] + "'");
        seen[d[1]] = d[0];
    }

    // WGSL allows @diagnostic on functions and control-flow statements only
    static void no_diagnostic(const Attrs &a) {
        if (const Attr *d = find_attr(a, "diagnostic")) invalid(d->line, d->col, "@diagnostic is allowed only on a function or a control-flow statement");
    }

    Attrs attrs() {
        Attrs out;
        std::map<std::string, std::string> diags;
        while (is("@")) {
            p++;
            Attr a;
            a.line = cur().line; a.col = cur().col;
            a.name = ident();
            if (a.name == "diagnostic") {   // checked, then ignored: there is no uniformity analysis to filter
                a.args = diagnostic_args();
                diagnostic_filter(diags, a.args, a.line, a.col);
            } else if (accept("(")) {
                while (!is(")")) {
                    if (cur().k == Tok::Id) a.args.push_back(t[p++].s);
                    else if (cur().k == Tok::Int) { a.args.push_back(std::to_string(t[p].iv)); p++; }
                    else err("unsupported attribute argument");
                    if (!accept(",")) break;
                }
                expect(")");
            }
            out.push_back(a);
        }
        return out;
    }

    TypeP type() {
        auto ty = std::make_shared<TypeExpr>();
        ty->line = cur().line; ty->col = cur().col;
        ty->name = ident();
        if (is("<")) {
            p++;
            while (!is(">")) {
                if (cur().k == Tok::Id && !(t[p + 1].k == Tok::Punct && (t[p + 1].s == "+" || t[p + 1].s == "*"))) {
                    ty->targs.push_back(type());
                    ty->eargs.push_back(nullptr);
                } else {
                    ty->targs.push_back(nullptr);
                    ty->eargs.push_back(expr_no_gt());
                }
                if (!accept(",")) break;
            }
            if (is(">>")) { t[p].s = ">"; }   // a nested list closed by '>>'
            else expect(">");
        }
        return ty;
    }

    bool no_gt = false;   // inside a template list: '>' ends it
    ExprP expr_no_gt() {
        bool s = no_gt;
        no_gt = true;
        ExprP e = expr();
        no_gt = s;
        return e;
    }

    ExprP mk(Expr::K k) {
        auto e = std::make_shared<Expr>();
        e->k = k; e->line = cur().line; e->col = cur().col;
        return e;
    }

    ExprP primary() {
        const Tok &tk = cur();
        if (tk.k == Tok::Int || tk.k == Tok::Float) {
            ExprP e = mk(Expr::Lit);
            e->lk = tk.k == Tok::Int ? 'i' : 'f';
            e->iv = tk.iv; e->fv = tk.fv; e->suf = tk.s;
            if (tk.k == Tok::Int && tk.s == "f") { e->lk = 'f'; e->fv = (double)tk.iv; }
            p++;
            return e;
        }
        if (tk.k == Tok::Id && (tk.s == "true" || tk.s == "false")) {
            ExprP e = mk(Expr::Lit);
            e->lk = 'b'; e->bv = tk.s == "true";
            p++;
            return e;
        }
        if (accept("(")) {
            bool s = no_gt;
            no_gt = false;
            ExprP e = expr();
            no_gt = s;
            expect(")");
            return e;
        }
        if (tk.k == Tok::Id) {
            ExprP e = mk(Expr::Id);
            bool templ = kTemplated.count(tk.s) && t[p + 1].k == Tok::Punct && t[p + 1].s == "<";
            if (templ || (t[p + 1].k == Tok::Punct && t[p + 1].s == "(")) {
                e->k = Expr::Call;
                e->callee = type();
                expect("(");
                bool s = no_gt;
                no_gt = false;
                while (!is(")")) {
                    e->a.push_back(expr());
                    if (!accept(",")) break;
                }
                no_gt = s;
                expect(")");
                return e;
            }
            e->s = ident();
            return e;
        }
        err("expected an expression, found '" + (tk.k == Tok::End ? std::string("end of file") : tk.s) + "'");
    }

    ExprP postfix(ExprP e) {
        for (;;) {
            if (is("[")) {
                ExprP x = mk(Expr::Idx);
                p++;
                bool s = no_gt;
                no_gt = false;
                x->a = {e, expr()};
                no_gt = s;
                expect("]");
                e = x;
            } else if (is(".")) {
                ExprP x = mk(Expr::Mem);
                p++;
                x->s = ident();
                x->a = {e};
                e = x;
            } else {
                return e;
            }
        }
    }

    ExprP unary() {
        if (is("-") || is("!") || is("~") || is("&") || is("*")) {
            ExprP e = mk(Expr::Un);
            e->s = t[p++].s;
            if (e->s == "&" || e->s == "*") unsupported(e->line, e->col, "pointers");
            e->a = {unary()};
            return e;
        }
        return postfix(primary());
    }

    int prec(const std::string &op) const {
        if (op == "||") return 1;
        if (op == "&&") return 2;
        if (op == "|") return 3;
        if (op == "^") return 4;
        if (op == "&") return 5;
        if (op == "==" || op == "!=") return 6;
        if (op == "<" || op == ">" || op == "<=" || op == ">=") return 7;
        if (op == "<<" || op == ">>") return 8;
        if (op == "+" || op == "-") return 9;
        if (op == "*" || op == "/" || op == "%") return 10;
        return 0;
    }
    ExprP binary(int min) {
        ExprP l = unary();
        for (;;) {
            if (cur().k != Tok::Punct) return l;
            std::string op = cur().s;
            if (no_gt && (op == ">" || op == ">>" || op == ">=")) return l;
            int pr = prec(op);
            if (pr == 0 || pr < min) return l;
            ExprP e = mk(Expr::Bin);
            p++;
            e->s = op;
            e->a = {l, binary(pr + 1)};
            l = e;
        }
    }
    ExprP expr() { return binary(1); }

    StmtP mks(Stmt::K k) {
        auto s = std::make_shared<Stmt>();
        s->k = k; s->line = cur().line; s->col = cur().col;
        return s;
    }

    std::vector<StmtP> block() {
        expect("{");
        std::vector<StmtP> out;
        while (!is("}")) {
            if (cur().k == Tok::End) err("expected '}'");
            out.push_back(stmt());
        }
        p++;
        return out;
    }

    // a statement that may appear in a for header: declaration, assignment, increment or call
    StmtP simple() {
        if (is_id("var") || is_id("let") || is_id("const")) {
            StmtP s = mks(cur().s == "var" ? Stmt::Var : cur().s == "let" ? Stmt::Let : Stmt::Const);
            p++;
            if (s->k == Stmt::Var && is("<")) unsupported(s->line, s->col, "address spaces on function-scope variables");
            s->name = ident();
            if (accept(":")) s->ty = type();
            if (accept("=")) s->e = expr();
            else if (s->k != Stmt::Var) err("a let or const declaration needs an initializer");
            return s;
        }
        if (is("_")) {
            StmtP s = mks(Stmt::Phony);
            p++;
            expect("=");
            s->e = expr();
            return s;
        }
        ExprP e = unary();
        if (is("++") || is("--")) {
            StmtP s = mks(is("++") ? Stmt::Incr : Stmt::Decr);
            p++;
            s->lhs = e;
            return s;
        }
        static const char *ops[] = {"=", "+=", "-=", "*=", "/=", "%=", "&=", "|=", "^=", "<<=", ">>="};
        for (const char *o : ops) {
            if (is(o)) {
                StmtP s = mks(Stmt::Assign);
                p++;
                s->op = o;
                s->lhs = e;
                s->e = expr();
                return s;
            }
        }
        if (e->k != Expr::Call) err("expected a statement");
        StmtP s = mks(Stmt::CallS);
        s->e = e;
        return s;
    }

    StmtP if_stmt() {
        StmtP s = mks(Stmt::If);
        p++;
        s->e = expr();
        s->body = block();
        if (is_id("else")) {
            p++;
            if (is_id("if")) s->els = if_stmt();
            else {
                s->els = mks(Stmt::Block);
                s->els->body = block();
            }
        }
        return s;
    }

    StmtP stmt() {
        Attrs a = attrs();
        if (!(is("{") || is_id("if") || is_id("switch") || is_id("loop") || is_id("for") || is_id("while"))) no_diagnostic(a);
        if (accept(";")) return mks(Stmt::Block);
        if (is("{")) {
            StmtP s = mks(Stmt::Block);
            s->body = block();
            return s;
        }
        if (is_id("if")) return if_stmt();
        if (is_id("switch")) {
            StmtP s = mks(Stmt::Switch);
            p++;
            s->e = expr();
            expect("{");
            while (!is("}")) {
                Clause c;
                if (is_id("default")) {
                    p++;
                    c.def = true;
                } else {
                    if (!is_id("case")) err("expected 'case' or 'default'");
                    p++;
                    while (!is(":") && !is("{")) {
                        if (is_id("default")) { p++; c.def = true; }
                        else c.sels.push_back(expr());
                        if (!accept(",")) break;
                    }
                }
                accept(":");
                c.body = block();
                s->clauses.push_back(c);
            }
            p++;
            return s;
        }
        if (is_id("loop")) {
            StmtP s = mks(Stmt::Loop);
            p++;
            expect("{");
            while (!is("}")) {
                if (is_id("continuing")) {
                    p++;
                    expect("{");
                    while (!is("}")) {
                        if (is_id("break") && t[p + 1].k == Tok::Id && t[p + 1].s == "if") {
                            StmtP b = mks(Stmt::BreakIf);
                            p += 2;
                            b->e = expr();
                            expect(";");
                            s->cont.push_back(b);
                        } else {
                            s->cont.push_back(stmt());
                        }
                    }
                    p++;
                    break;
                }
                s->body.push_back(stmt());
            }
            expect("}");
            return s;
        }
        if (is_id("for")) {
            StmtP s = mks(Stmt::For);
            p++;
            expect("(");
            if (!is(";")) s->init = simple();
            expect(";");
            if (!is(";")) s->e = expr();
            expect(";");
            if (!is(")")) s->update = simple();
            expect(")");
            s->body = block();
            return s;
        }
        if (is_id("while")) {
            StmtP s = mks(Stmt::While);
            p++;
            s->e = expr();
            s->body = block();
            return s;
        }
        StmtP s;
        if (is_id("break")) { s = mks(Stmt::Break); p++; }
        else if (is_id("continue")) { s = mks(Stmt::Continue); p++; }
        else if (is_id("discard")) { s = mks(Stmt::Discard); p++; }
        else if (is_id("return")) {
            s = mks(Stmt::Return);
            p++;
            if (!is(";")) s->e = expr();
        } else if (is_id("const_assert")) {
            s = const_assert();
        } else {
            s = simple();
        }
        expect(";");
        return s;
    }

    StmtP const_assert() {
        StmtP s = mks(Stmt::ConstAssert);
        p++;
        s->e = expr();
        return s;
    }

    void module() {
        bool declared = false;   // directives come before every declaration
        while (cur().k != Tok::End) {
            if (accept(";")) continue;
            if (is_id("diagnostic")) {
                int line = cur().line, col = cur().col;
                if (declared) invalid(line, col, "a diagnostic directive must come before every declaration");
                p++;
                diagnostic_filter(module_diagnostics, diagnostic_args(), line, col);
                expect(";");
                continue;
            }
            declared = declared || !is_id("enable");
            if (is_id("const_assert")) {
                m.asserts.push_back(const_assert());
                expect(";");
                continue;
            }
            if (is_id("enable")) {
                p++;
                for (;;) {
                    std::string ext = ident();
                    if (ext != "wgpu_binding_array") unsupported(t[p - 1].line, t[p - 1].col, "enable " + ext);
                    if (!accept(",")) break;
                }
                expect(";");
                continue;
            }
            if (is_id("requires")) unsupported(cur().line, cur().col, "requires directives");
            Attrs a = attrs();
            int line = cur().line, col = cur().col;
            if (!is_id("fn")) no_diagnostic(a);
            if (is_id("struct")) {
                p++;
                StructDecl s;
                s.line = line; s.col = col;
                s.name = ident();
                expect("{");
                while (!is("}")) {
                    Member mb;
                    mb.attrs = attrs();
                    no_diagnostic(mb.attrs);
                    mb.line = cur().line; mb.col = cur().col;
                    mb.name = ident();
                    expect(":");
                    mb.ty = type();
                    s.members.push_back(mb);
                    if (!accept(",")) break;
                }
                expect("}");
                accept(";");
                m.structs.push_back(s);
            } else if (is_id("var")) {
                p++;
                Global g;
                g.line = line; g.col = col;
                g.attrs = a;
                if (accept("<")) {
                    g.space = ident();
                    if (accept(",")) g.access = ident();
                    expect(">");
                }
                g.name = ident();
                if (accept(":")) g.ty = type();
                if (accept("=")) g.init = expr();
                expect(";");
                m.globals.push_back(g);
            } else if (is_id("const")) {
                p++;
                ConstDecl c;
                c.line = line; c.col = col;
                c.name = ident();
                if (accept(":")) c.ty = type();
                expect("=");
                c.init = expr();
                expect(";");
                m.consts.push_back(c);
            } else if (is_id("override")) {
                unsupported(line, col, "override declarations");
            } else if (is_id("alias")) {
                p++;
                AliasDecl a;
                a.line = line; a.col = col;
                a.name = ident();
                expect("=");
                a.ty = type();
                expect(";");
                m.aliases.push_back(a);
            } else if (is_id("fn")) {
                p++;
                FnDecl f;
                f.line = line; f.col = col;
                f.attrs = a;
                f.name = ident();
                expect("(");
                while (!is(")")) {
                    Param pr;
                    pr.attrs = attrs();
                    no_diagnostic(pr.attrs);
                    pr.line = cur().line; pr.col = cur().col;
                    pr.name = ident();
                    expect(":");
                    pr.ty = type();
                    f.params.push_back(pr);
                    if (!accept(",")) break;
                }
                expect(")");
                if (accept("->")) {
                    f.ret_attrs = attrs();
                    no_diagnostic(f.ret_attrs);
                    f.ret = type();
                }
                f.body = block();
                m.fns.push_back(f);
            } else {
                err("expected a declaration");
            }
        }
    }
};

// --------------------------------------------------------------------------------------------------------------- checker
struct FieldInfo {
    std::string name;
    Ty ty;
    Attrs attrs;
    uint32_t offset = 0;
    uint32_t size = 0, align = 0;   // @size / @align, 0 when absent
};
struct StructInfo {
    std::string name;
    std::vector<FieldInfo> fields;
    int line = 0, col = 0;
    bool resolved = false;
    std::string cname;   // a predeclared result struct (frexp, modf): its wgsl_rt.cuh type
};

// a const-expression's value, as const_assert evaluates it: s the scalar kind, n 0 (a scalar) or the vector size; floats
// in f, integers and bools in i
struct KV {
    SK s = S_BOOL;
    int n = 0;
    double f[4] = {0, 0, 0, 0};
    long long i[4] = {0, 0, 0, 0};
};

struct Sym {
    enum K { Local, Param, Const, ModConst, Uniform, Base, Textures, Sampler, Private } k = Local;
    Ty ty;
    bool mut = false;
    bool has_cv = false;
    CV cv;
    std::string code;
    bool cint = false;   // a constant of concrete integer type, whose value is civ
    long long civ = 0;
    bool is_const = false;       // a const declaration: kv is its value when kv_status is 0
    int kv_status = 0;           // otherwise why it has none (SMR_ERR_INVALID_ARGUMENT: not a const-expression)
    KV kv;
};

struct FnInfo {
    const FnDecl *d;
    std::vector<Ty> params;
    Ty ret;
    std::string cname;
    std::vector<std::string> calls;   // the user functions it calls
    int frag_line = 0, frag_col = 0;  // its first fragment-only builtin, if any
};

const char *kUnsupportedFns[] = {"dpdx", "dpdy", "fwidth", "dpdxCoarse", "dpdyCoarse", "dpdxFine", "dpdyFine", "fwidthCoarse",
                                 "fwidthFine", "atomicLoad", "atomicStore", "atomicAdd", "atomicSub", "atomicMax", "atomicMin",
                                 "atomicAnd", "atomicOr", "atomicXor", "atomicExchange", "atomicCompareExchangeWeak",
                                 "textureLoad", "textureSampleCompare", "textureSampleCompareLevel", "textureGatherCompare",
                                 "textureStore", "textureNumLayers", "textureNumSamples", "arrayLength", "workgroupBarrier",
                                 "storageBarrier", "textureBarrier", "workgroupUniformLoad", "subgroupAdd",
                                 "subgroupBroadcast", "f16", "ptr", "atomic"};
// the texture builtins: their texture and sampler arguments are checked where they are translated
const std::set<std::string> kTextureFns = {"textureSample", "textureSampleLevel", "textureSampleBias", "textureSampleGrad",
                                           "textureSampleBaseClampToEdge", "textureGather", "textureDimensions",
                                           "textureNumLevels"};

struct Checker {
    Module &m;
    std::vector<StructInfo> structs;
    std::map<std::string, int> struct_ids;
    std::vector<std::map<std::string, Sym>> scopes;
    std::map<std::string, FnInfo> fns;
    std::string out_structs, out_consts, out_loaders, out_protos, out_bodies;
    FnInfo *cur_fn = nullptr;
    std::string cur_stage;            // "vertex", "fragment" or "" (a helper)
    std::vector<int> loops;           // label numbers of the enclosing loops (-1: a switch)
    int label = 0;
    const Global *uniform = nullptr;
    Ty uniform_ty;
    std::map<std::string, std::string> loader_names;
    std::map<std::string, const AliasDecl *> aliases;
    std::string out_private, out_private_init;   // var<private>: the members of wg_private and their initialisers
    std::vector<std::string> alias_stack;   // the aliases being resolved, to find a cycle

    explicit Checker(Module &mod) : m(mod) {}

    // ---- types ----
    std::string sname(SK s) const {
        switch (s) {
            case S_BOOL: return "bool";
            case S_I32: return "i32";
            case S_U32: return "u32";
            case S_F32: return "f32";
            case S_AI: return "abstract-int";
            default: return "abstract-float";
        }
    }
    std::string tname(const Ty &t) const {
        switch (t.k) {
            case Ty::Void: return "void";
            case Ty::Scalar: return sname(t.s);
            case Ty::Vec: return "vec" + std::to_string(t.n) + "<" + sname(t.s) + ">";
            case Ty::Mat: return "mat" + std::to_string(t.n) + "x" + std::to_string(t.m) + "<f32>";
            case Ty::Arr: return "array<" + tname(*t.el) + ", " + std::to_string(t.n) + ">";
            case Ty::Struct: return structs[t.sid].name;
            case Ty::Tex: return "texture_2d<f32>";
            case Ty::Samp: return "sampler";
            default: return "binding_array<texture_2d<f32>, " + std::to_string(t.n) + ">";
        }
    }
    std::string cscalar(SK s) const {
        switch (concrete_of(s)) {
            case S_BOOL: return "bool";
            case S_I32: return "int";
            case S_U32: return "unsigned";
            default: return "float";
        }
    }
    std::string cty(const Ty &t) const {
        switch (t.k) {
            case Ty::Scalar: return cscalar(t.s);
            case Ty::Vec: return "wv<" + cscalar(t.s) + ", " + std::to_string(t.n) + ">";
            case Ty::Mat: return "wm<" + std::to_string(t.n) + ", " + std::to_string(t.m) + ">";
            case Ty::Arr: return "wa<" + cty(*t.el) + ", " + std::to_string(t.n) + ">";
            case Ty::Struct: return structs[t.sid].cname.empty() ? "S_" + structs[t.sid].name : structs[t.sid].cname;
            case Ty::Tex: return "unsigned";      // a texture value is its binding-array index
            case Ty::Samp: return "wg_sampler";
            default: return "void";
        }
    }

    long long const_int(const ExprP &e) {
        Ty t = check(e);
        if (!e->has_cv || e->cv.f || e->cv.n) {
            if (e->k == Expr::Id) unsupported(e->line, e->col, "array sizes that are not constant integers");
            invalid(e->line, e->col, "expected a constant integer");
        }
        (void)t;
        return e->cv.iv[0];
    }

    SK scalar_kind(const TypeP &tp) {
        Ty t = resolve(tp);
        if (t.k != Ty::Scalar) invalid(tp->line, tp->col, "expected a scalar type");
        return t.s;
    }

    Ty resolve(const TypeP &tp) {
        const std::string &n = tp->name;
        auto al = aliases.find(n);
        if (al != aliases.end()) {   // a type alias is its target, wherever it is written
            if (!tp->targs.empty()) invalid(tp->line, tp->col, "the alias " + n + " takes no template arguments");
            for (const std::string &a : alias_stack) if (a == n) invalid(al->second->line, al->second->col, "alias " + n + " refers to itself");
            alias_stack.push_back(n);
            Ty t = resolve(al->second->ty);
            alias_stack.pop_back();
            return t;
        }
        auto need = [&](size_t k) {
            if (tp->targs.size() != k) invalid(tp->line, tp->col, n + " expects " + std::to_string(k) + " template argument(s)");
        };
        auto targ = [&](size_t i) -> const TypeP & {
            if (!tp->targs[i]) invalid(tp->line, tp->col, "expected a type argument");
            return tp->targs[i];
        };
        if (n == "f32" || n == "i32" || n == "u32" || n == "bool") {
            need(0);
            return scalar(n == "f32" ? S_F32 : n == "i32" ? S_I32 : n == "u32" ? S_U32 : S_BOOL);
        }
        if (n == "f16") unsupported(tp->line, tp->col, "f16");
        if (n.size() == 4 && n.compare(0, 3, "vec") == 0 && n[3] >= '2' && n[3] <= '4') {
            need(1);
            SK s = scalar_kind(targ(0));
            return vec(s, n[3] - '0');
        }
        if (n.size() == 6 && n.compare(0, 3, "mat") == 0 && n[4] == 'x' && n[3] >= '2' && n[3] <= '4' && n[5] >= '2' && n[5] <= '4') {
            need(1);
            if (scalar_kind(targ(0)) != S_F32) unsupported(tp->line, tp->col, "matrices of other than f32");
            Ty t;
            t.k = Ty::Mat; t.n = n[3] - '0'; t.m = n[5] - '0';
            return t;
        }
        if ((n.size() == 6 && n[0] == 'v' && n.compare(0, 3, "vec") == 0 && n[4] == 'f') || n == "vec2f" || n == "vec3f" ||
            n == "vec4f" || n == "vec2i" || n == "vec3i" || n == "vec4i" || n == "vec2u" || n == "vec3u" || n == "vec4u") {
            need(0);
            return vec(n[4] == 'f' ? S_F32 : n[4] == 'i' ? S_I32 : S_U32, n[3] - '0');
        }
        if (n == "vec2h" || n == "vec3h" || n == "vec4h") unsupported(tp->line, tp->col, "f16");
        if (n.size() == 7 && n.compare(0, 3, "mat") == 0 && n[4] == 'x' && n[6] == 'f') {
            need(0);
            Ty t;
            t.k = Ty::Mat; t.n = n[3] - '0'; t.m = n[5] - '0';
            if (t.n < 2 || t.n > 4 || t.m < 2 || t.m > 4) invalid(tp->line, tp->col, "unknown type " + n);
            return t;
        }
        if (n == "array") {
            if (tp->targs.size() == 1) unsupported(tp->line, tp->col, "runtime-sized arrays");
            need(2);
            Ty el = resolve(targ(0));
            size_expr(tp);
            long long len = const_int(tp->eargs[1]);
            if (len <= 0 || len > (1 << 16)) invalid(tp->line, tp->col, "array length out of range");
            Ty t;
            t.k = Ty::Arr; t.el = std::make_shared<Ty>(el); t.n = (int)len;
            return t;
        }
        if (n == "binding_array") {
            need(2);
            Ty el = resolve(targ(0));
            if (el.k != Ty::Tex) unsupported(tp->line, tp->col, "binding arrays of other than texture_2d<f32>");
            size_expr(tp);
            long long len = const_int(tp->eargs[1]);
            Ty t;
            t.k = Ty::TexArr; t.n = (int)len;
            return t;
        }
        if (n == "texture_2d") {
            need(1);
            if (scalar_kind(targ(0)) != S_F32) unsupported(tp->line, tp->col, "texture_2d<" + targ(0)->name + ">");
            Ty t;
            t.k = Ty::Tex;
            return t;
        }
        if (n == "sampler") { Ty t; t.k = Ty::Samp; return t; }
        if (n.compare(0, 8, "texture_") == 0 || n == "sampler_comparison") unsupported(tp->line, tp->col, "textures other than the header's (" + n + ")");
        if (n == "ptr") unsupported(tp->line, tp->col, "pointers");
        if (n == "atomic") unsupported(tp->line, tp->col, "atomics");
        auto it = struct_ids.find(n);
        if (it != struct_ids.end()) {
            resolve_struct(it->second);
            Ty t;
            t.k = Ty::Struct; t.sid = it->second;
            return t;
        }
        invalid(tp->line, tp->col, "unknown type '" + n + "'");
    }

    // an array size written as an identifier (a constant) parses as a type
    void size_expr(const TypeP &tp) {
        if (tp->eargs[1] || !tp->targs[1]) return;
        auto e = std::make_shared<Expr>();
        e->k = Expr::Id; e->s = tp->targs[1]->name; e->line = tp->targs[1]->line; e->col = tp->targs[1]->col;
        tp->eargs[1] = e;
    }

    std::vector<int> resolving;
    void resolve_struct(int id) {
        StructInfo &si = structs[id];
        if (si.resolved) return;
        for (int r : resolving) if (r == id) invalid(si.line, si.col, "struct " + si.name + " contains itself");
        resolving.push_back(id);
        const StructDecl *d = nullptr;
        for (const StructDecl &s : m.structs) if (s.name == si.name) d = &s;
        std::string body = "struct S_" + si.name + " {\n";
        std::set<std::string> seen;
        for (const Member &mb : d->members) {
            if (!seen.insert(mb.name).second) invalid(mb.line, mb.col, "duplicate member " + mb.name);
            for (const Attr &a : mb.attrs) {
                if (a.name == "builtin" && !a.args.empty() && a.args[0] != "position" && a.args[0] != "front_facing")
                    unsupported(a.line, a.col, "@builtin(" + a.args[0] + ")");
            }
            FieldInfo f;
            f.name = mb.name;
            f.ty = resolve(mb.ty);
            if (f.ty.k == Ty::Tex || f.ty.k == Ty::Samp || f.ty.k == Ty::TexArr) invalid(mb.line, mb.col, "a struct member cannot be a texture or sampler");
            f.attrs = mb.attrs;
            for (const Attr &a : mb.attrs) {   // @size / @align: the member's place in memory (the uniform's layout)
                if (a.name != "size" && a.name != "align") continue;
                uint32_t ta, ts;
                layout(f.ty, ta, ts, a.line, a.col, false);
                const long long v = attr_int(a);
                if (a.name == "align") {
                    if (v <= 0 || (v & (v - 1)) || v > (1LL << 30)) invalid(a.line, a.col, "@align must be a positive power of two, found " + std::to_string(v));
                    // a member sits at a multiple of its type's alignment in every address space (RequiredAlignOf)
                    if (v < (long long)ta) invalid(a.line, a.col, "@align(" + std::to_string(v) + ") is below the AlignOf " + std::to_string(ta) + " of " + tname(f.ty));
                    f.align = (uint32_t)v;
                } else {
                    if (v < (long long)ts || v > (1LL << 30)) invalid(a.line, a.col, "@size(" + std::to_string(v) + ") is below the SizeOf " + std::to_string(ts) + " of " + tname(f.ty));
                    f.size = (uint32_t)v;
                }
            }
            si.fields.push_back(f);
            body += "    " + cty(f.ty) + " m_" + mb.name + ";\n";
        }
        body += "};\n";
        out_structs += body;
        si.resolved = true;
        resolving.pop_back();
    }

    // an attribute's one integer argument: a literal or a module constant
    long long attr_int(const Attr &a) {
        if (a.args.size() != 1) invalid(a.line, a.col, "@" + a.name + " takes one argument");
        const std::string &v = a.args[0];
        if (isdigit((unsigned char)v[0])) return atoll(v.c_str());
        Sym *s = lookup(v);
        if (s && s->k == Sym::ModConst && s->has_cv && !s->cv.f && !s->cv.n) return s->cv.iv[0];
        if (s && s->k == Sym::ModConst && s->cint) return s->civ;
        invalid(a.line, a.col, "@" + a.name + " needs a constant integer");
    }

    // WGSL's memory layout (AlignOf, SizeOf, array stride; a member's @align / @size replace its type's); `uniform`: with
    // the uniform address space's constraints checked
    void layout(const Ty &t, uint32_t &align, uint32_t &size, int line, int col, bool uniform = true) {
        switch (t.k) {
            case Ty::Scalar:
                if (uniform && t.s == S_BOOL) invalid(line, col, "bool is not host-shareable and cannot be in a uniform");
                align = size = 4;
                return;
            case Ty::Vec:
                if (uniform && t.s == S_BOOL) invalid(line, col, "bool is not host-shareable and cannot be in a uniform");
                align = t.n == 2 ? 8 : 16;
                size = 4 * t.n;
                return;
            case Ty::Mat: {
                uint32_t ca = t.m == 2 ? 8 : 16;
                align = ca;
                size = ca * t.n;
                return;
            }
            case Ty::Arr: {
                uint32_t ea, es;
                layout(*t.el, ea, es, line, col, uniform);
                uint32_t stride = (es + ea - 1) / ea * ea;
                if (uniform && stride % 16) invalid(line, col, "the uniform address space needs an array stride that is a multiple of 16; " +
                                                    tname(t) + " has " + std::to_string(stride));
                align = ea;
                size = stride * t.n;
                return;
            }
            case Ty::Struct: {
                StructInfo &si = structs[t.sid];
                uint32_t off = 0, al = 1;
                bool after_struct = false;
                uint32_t min_next = 0;
                for (FieldInfo &f : si.fields) {
                    uint32_t ta, ts;
                    layout(f.ty, ta, ts, line, col, uniform);
                    const uint32_t fa = f.align ? f.align : ta, fs = f.size ? f.size : ts;
                    off = (off + fa - 1) / fa * fa;
                    if (uniform && (f.ty.k == Ty::Struct || f.ty.k == Ty::Arr) && off % 16)
                        invalid(line, col, "the uniform address space needs member " + si.name + "." + f.name + " at a multiple of 16");
                    if (uniform && after_struct && off < min_next)
                        invalid(line, col, "the uniform address space needs 16 bytes of padding after a struct member of " + si.name);
                    f.offset = off;
                    after_struct = f.ty.k == Ty::Struct;
                    min_next = off + (ts + 15) / 16 * 16;
                    off += fs;
                    al = std::max(al, fa);
                }
                align = al;
                size = (off + al - 1) / al * al;
                return;
            }
            default:
                invalid(line, col, "a uniform cannot hold " + tname(t));
        }
    }

    // code that loads a value of type t from the parameter bytes at `p`
    std::string load(const Ty &t, const std::string &p) {
        switch (t.k) {
            case Ty::Scalar: return "wld<" + cscalar(t.s) + ">(" + p + ")";
            case Ty::Vec: return "wldv<" + cscalar(t.s) + ", " + std::to_string(t.n) + ">(" + p + ")";
            default: {
                std::string key = cty(t);
                auto it = loader_names.find(key);
                if (it != loader_names.end()) return it->second + "(" + p + ")";
                std::string body;   // the members' loaders first: they take their names before this one

                if (t.k == Ty::Mat) {
                    uint32_t cs = t.m == 2 ? 8 : 16;
                    for (int c = 0; c < t.n; c++)
                        body += "    r.c[" + std::to_string(c) + "] = wldv<float, " + std::to_string(t.m) + ">(p + " + std::to_string(c * cs) + ");\n";
                } else if (t.k == Ty::Arr) {
                    uint32_t ea, es;
                    layout(*t.el, ea, es, 0, 0);
                    uint32_t stride = (es + ea - 1) / ea * ea;
                    body += "    for (int i = 0; i < " + std::to_string(t.n) + "; i++) r.a[i] = " + load(*t.el, "p + " + std::to_string(stride) + " * i") + ";\n";
                } else {
                    for (const FieldInfo &f : structs[t.sid].fields) body += "    r.m_" + f.name + " = " + load(f.ty, "p + " + std::to_string(f.offset)) + ";\n";
                }
                body += "    return r;\n}\n";
                std::string name = "wl_" + std::to_string(loader_names.size());
                out_loaders += "__device__ inline " + key + " " + name + "(const unsigned char *p) {\n    " + key + " r;\n" + body;
                loader_names[key] = name;
                return name + "(" + p + ")";
            }
        }
    }

    // ---- abstract values ----
    std::string lit(const CV &cv, int i, SK to, int line, int col) {
        char buf[64];
        if (to == S_F32 || to == S_AF) {
            double d = cv.f ? cv.fv[i] : (double)cv.iv[i];
            float f = (float)d;
            if (!std::isfinite(f)) invalid(line, col, "value out of the range of f32");
            snprintf(buf, sizeof buf, "%.9ef", (double)f);
            return buf;
        }
        if (cv.f) invalid(line, col, "cannot convert an abstract float to " + sname(to));
        long long v = cv.iv[i];
        if (to == S_I32 || to == S_AI) {
            if (v < -2147483648ll || v > 2147483647ll) invalid(line, col, "value " + std::to_string(v) + " out of the range of i32");
            if (v == -2147483648ll) return "(-2147483647 - 1)";
            return std::to_string(v);
        }
        if (to == S_U32) {
            if (v < 0 || v > 4294967295ll) invalid(line, col, "value " + std::to_string(v) + " out of the range of u32");
            return std::to_string(v) + "u";
        }
        invalid(line, col, "cannot convert a number to bool");
    }

    // can an expression of type `from` take type `to` (the same type, or abstract converted)?
    static bool convertible(SK from, SK to) {
        if (from == to) return true;
        if (from == S_AI) return to == S_I32 || to == S_U32 || to == S_F32 || to == S_AF;
        if (from == S_AF) return to == S_F32;
        return false;
    }
    void conv(const ExprP &e, const Ty &to) {
        const Ty &t = e->ty;
        bool ok = t == to;
        if (!ok && abstract(t) && (t.k == to.k) && t.n == to.n && to.k != Ty::Mat) ok = convertible(t.s, to.s);
        if (!ok) invalid(e->line, e->col, "expected " + tname(to) + ", found " + tname(t));
        if (abstract(t)) { e->has_target = true; e->target = to; }
    }
    void conv_default(const ExprP &e) {
        if (abstract(e->ty)) conv(e, concrete(e->ty));
    }
    // the common element kind of two numeric kinds, or an error
    SK unify(SK a, SK b, const ExprP &at) {
        if (a == b) return a;
        if (convertible(a, b)) return b;
        if (convertible(b, a)) return a;
        invalid(at->line, at->col, "mismatched operand types " + sname(a) + " and " + sname(b));
    }

    // a const of concrete integer type keeps its value, for the builtins that need a const-expression (textureGather)
    void const_int(Sym &sym, const ExprP &init) {
        if (sym.ty.k != Ty::Scalar || !integral(sym.ty.s)) return;
        if (init->has_cv && !init->cv.f && !init->cv.n) { sym.cint = true; sym.civ = init->cv.iv[0]; }
        else if (init->cint) { sym.cint = true; sym.civ = init->civ; }
    }

    // ---- expressions ----
    Ty set(const ExprP &e, const Ty &t) { e->ty = t; return t; }
    Ty set_cv(const ExprP &e, const CV &cv) {
        e->has_cv = true;
        e->cv = cv;
        return set(e, cv.n ? vec(cv.f ? S_AF : S_AI, cv.n) : scalar(cv.f ? S_AF : S_AI));
    }

    Sym *lookup(const std::string &n) {
        for (auto it = scopes.rbegin(); it != scopes.rend(); ++it) {
            auto f = it->find(n);
            if (f != it->end()) return &f->second;
        }
        return nullptr;
    }

    Ty check(const ExprP &e) {
        switch (e->k) {
            case Expr::Lit: {
                if (e->lk == 'b') { e->code = e->bv ? "true" : "false"; return set(e, scalar(S_BOOL)); }
                CV cv;
                cv.f = e->lk == 'f';
                cv.fv[0] = e->fv;
                cv.iv[0] = e->iv;
                if (e->suf.empty()) return set_cv(e, cv);
                SK s = e->suf == "f" ? S_F32 : e->suf == "i" ? S_I32 : S_U32;   // a suffixed literal is concrete
                e->code = lit(cv, 0, s, e->line, e->col);
                e->cint = s != S_F32;
                e->civ = e->iv;
                return set(e, scalar(s));
            }
            case Expr::Id: {
                Sym *s = lookup(e->s);
                if (!s) {
                    for (const char *u : kUnsupportedFns) if (e->s == u) unsupported(e->line, e->col, e->s);
                    invalid(e->line, e->col, "unknown identifier '" + e->s + "'");
                }
                if (s->has_cv) { e->has_cv = true; e->cv = s->cv; return set(e, s->ty); }
                e->code = s->code;
                e->uref = s->k == Sym::Uniform;
                e->cint = s->cint;
                e->civ = s->civ;
                return set(e, s->ty);
            }
            case Expr::Un: return check_unary(e);
            case Expr::Bin: return check_binary(e);
            case Expr::Call: return check_call(e);
            case Expr::Idx: return check_index(e);
            case Expr::Mem: return check_member(e);
        }
        return Ty();
    }

    // a value's code once its type is fixed: an abstract value as a literal of its target type
    std::string code(const ExprP &e) {
        if (e->uref) return load(e->ty, "ctx.params + " + e->code);
        if (!e->has_cv) return e->code;
        Ty to = e->has_target ? e->target : concrete(e->ty);
        if (to.k == Ty::Scalar) return lit(e->cv, 0, to.s, e->line, e->col);
        std::string s = cty(to) + "{{";
        for (int i = 0; i < to.n; i++) s += (i ? ", " : "") + lit(e->cv, i, to.s, e->line, e->col);
        return s + "}}";
    }

    Ty check_unary(const ExprP &e) {
        Ty t = check(e->a[0]);
        const std::string &op = e->s;
        if (op == "!") {
            if (!(t.k == Ty::Scalar || t.k == Ty::Vec) || t.s != S_BOOL) invalid(e->line, e->col, "'!' needs bool, found " + tname(t));
            e->code = "w_lnot(" + code(e->a[0]) + ")";
            return set(e, t);
        }
        if (!(t.k == Ty::Scalar || t.k == Ty::Vec) || !numeric(t.s)) invalid(e->line, e->col, "'" + op + "' needs a number, found " + tname(t));
        if (op == "-") {
            if (e->a[0]->has_cv) {
                CV cv = e->a[0]->cv;
                for (int i = 0; i < 4; i++) { cv.fv[i] = -cv.fv[i]; cv.iv[i] = -cv.iv[i]; }
                return set_cv(e, cv);
            }
            if (t.s == S_U32) invalid(e->line, e->col, "'-' cannot negate u32");
            e->code = "w_neg(" + code(e->a[0]) + ")";
            return set(e, t);
        }
        // '~'
        if (!integral(t.s)) invalid(e->line, e->col, "'~' needs an integer, found " + tname(t));
        conv_default(e->a[0]);
        t = concrete(t);
        e->code = "w_bnot(" + code(e->a[0]) + ")";
        return set(e, t);
    }

    bool fold(const std::string &op, const CV &a, const CV &b, CV &r, const ExprP &e) {
        if (a.n && b.n && a.n != b.n) return false;
        r = CV();
        r.f = a.f || b.f;
        r.n = std::max(a.n, b.n);
        for (int i = 0; i < std::max(1, r.n); i++) {
            int ia = a.n ? i : 0, ib = b.n ? i : 0;
            if (r.f) {
                double x = a.f ? a.fv[ia] : (double)a.iv[ia], y = b.f ? b.fv[ib] : (double)b.iv[ib];
                if (op == "+") r.fv[i] = x + y;
                else if (op == "-") r.fv[i] = x - y;
                else if (op == "*") r.fv[i] = x * y;
                else if (op == "/") r.fv[i] = x / y;
                else if (op == "%") r.fv[i] = x - y * std::trunc(x / y);
                else return false;
                if (!std::isfinite(r.fv[i])) invalid(e->line, e->col, "constant expression overflows");
            } else {
                long long x = a.iv[ia], y = b.iv[ib];
                __int128 v;
                if (op == "+") v = (__int128)x + y;
                else if (op == "-") v = (__int128)x - y;
                else if (op == "*") v = (__int128)x * y;
                else if (op == "/" || op == "%") {
                    if (y == 0) invalid(e->line, e->col, "integer division by zero in a constant expression");
                    v = op == "/" ? (__int128)x / y : (__int128)x % y;
                } else return false;
                if (v > (__int128)0x7fffffffffffffffll || v < -(__int128)0x7fffffffffffffffll - 1) invalid(e->line, e->col, "constant expression overflows");
                r.iv[i] = (long long)v;
            }
        }
        return true;
    }

    Ty check_binary(const ExprP &e) {
        const std::string &op = e->s;
        Ty L = check(e->a[0]), R = check(e->a[1]);
        const ExprP &a = e->a[0], &b = e->a[1];
        auto numv = [](const Ty &t) { return (t.k == Ty::Scalar || t.k == Ty::Vec) && numeric(t.s); };
        if (op == "&&" || op == "||") {
            if (L != scalar(S_BOOL) || R != scalar(S_BOOL)) invalid(e->line, e->col, "'" + op + "' needs bool operands");
            e->code = "(" + code(a) + " " + op + " " + code(b) + ")";
            return set(e, L);
        }
        static const std::map<std::string, std::string> fn = {{"+", "w_add"}, {"-", "w_sub"}, {"*", "w_mul"}, {"/", "w_div"},
                                                               {"%", "w_mod"}, {"==", "w_eq"}, {"!=", "w_ne"}, {"<", "w_lt"},
                                                               {"<=", "w_le"}, {">", "w_gt"}, {">=", "w_ge"}, {"&", "w_and"},
                                                               {"|", "w_or"}, {"^", "w_xor"}, {"<<", "w_shl"}, {">>", "w_shr"}};
        const std::string &f = fn.at(op);
        bool arith = op == "+" || op == "-" || op == "*" || op == "/" || op == "%";
        if (arith && (L.k == Ty::Mat || R.k == Ty::Mat)) {
            Ty r;
            auto f32 = [&](const ExprP &x) { if (x->ty.k == Ty::Scalar || x->ty.k == Ty::Vec) conv(x, with_elem(x->ty, S_F32)); };
            f32(a); f32(b);
            L = a->ty.k == Ty::Scalar || a->ty.k == Ty::Vec ? with_elem(L, S_F32) : L;
            R = b->ty.k == Ty::Scalar || b->ty.k == Ty::Vec ? with_elem(R, S_F32) : R;
            if ((op == "+" || op == "-") && L == R) r = L;
            else if (op == "*" && L.k == Ty::Mat && R == scalar(S_F32)) r = L;
            else if (op == "*" && R.k == Ty::Mat && L == scalar(S_F32)) r = R;
            else if (op == "*" && L.k == Ty::Mat && R.k == Ty::Vec && R.n == L.n) r = vec(S_F32, L.m);
            else if (op == "*" && R.k == Ty::Mat && L.k == Ty::Vec && L.n == R.m) r = vec(S_F32, R.n);
            else if (op == "*" && L.k == Ty::Mat && R.k == Ty::Mat && L.n == R.m) { r = L; r.n = R.n; }
            else invalid(e->line, e->col, "no '" + op + "' for " + tname(L) + " and " + tname(R));
            e->code = ordered(f, {code(a), code(b)});
            return set(e, r);
        }
        if (!(L.k == Ty::Scalar || L.k == Ty::Vec) || !(R.k == Ty::Scalar || R.k == Ty::Vec))
            invalid(e->line, e->col, "no '" + op + "' for " + tname(L) + " and " + tname(R));
        if (op == "<<" || op == ">>") {
            if (!integral(L.s) || !integral(R.s) || L.k != R.k || L.n != R.n) invalid(e->line, e->col, "no '" + op + "' for " + tname(L) + " and " + tname(R));
            conv_default(a);
            conv(b, with_elem(R, S_U32));
            e->code = ordered(f, {code(a), code(b)});
            return set(e, concrete(L));
        }
        if (op == "&" || op == "|" || op == "^") {
            if (L.k != R.k || L.n != R.n) invalid(e->line, e->col, "no '" + op + "' for " + tname(L) + " and " + tname(R));
            SK s = unify(L.s, R.s, e);
            if (!(integral(s) || (s == S_BOOL && op != "^"))) invalid(e->line, e->col, "no '" + op + "' for " + tname(L));
            Ty t = concrete(with_elem(L, s));
            conv(a, t); conv(b, t);
            e->code = ordered(f, {code(a), code(b)});
            return set(e, t);
        }
        bool cmp = !arith;
        if (arith && (!numv(L) || !numv(R))) invalid(e->line, e->col, "no '" + op + "' for " + tname(L) + " and " + tname(R));
        if (cmp && (L.k != R.k || L.n != R.n)) invalid(e->line, e->col, "no '" + op + "' for " + tname(L) + " and " + tname(R));
        if (cmp && (op != "==" && op != "!=") && (L.s == S_BOOL || R.s == S_BOOL)) invalid(e->line, e->col, "no '" + op + "' for bool");
        if (arith && a->has_cv && b->has_cv) {
            CV r;
            if (fold(op, a->cv, b->cv, r, e)) return set_cv(e, r);
        }
        if (L.k == Ty::Vec && R.k == Ty::Vec && L.n != R.n) invalid(e->line, e->col, "no '" + op + "' for " + tname(L) + " and " + tname(R));
        SK s = concrete_of(unify(L.s, R.s, e));
        conv(a, with_elem(L, s));
        conv(b, with_elem(R, s));
        std::string ca = code(a), cb = code(b);
        int n = std::max(L.k == Ty::Vec ? L.n : 0, R.k == Ty::Vec ? R.n : 0);
        if (L.k == Ty::Scalar && n) ca = "wsplat<" + std::to_string(n) + ">(" + ca + ")";
        if (R.k == Ty::Scalar && n) cb = "wsplat<" + std::to_string(n) + ">(" + cb + ")";
        e->code = ordered(f, {ca, cb});
        SK rs = cmp ? S_BOOL : s;
        return set(e, n ? vec(rs, n) : scalar(rs));
    }

    Ty check_index(const ExprP &e) {
        const ExprP &b = e->a[0], &i = e->a[1];
        Ty B = check(b), I = check(i);
        if (I.k != Ty::Scalar || !integral(I.s)) invalid(i->line, i->col, "an index must be i32 or u32, found " + tname(I));
        if (abstract(B)) { conv_default(b); B = concrete(B); }
        int n = B.k == Ty::Vec || B.k == Ty::Mat || B.k == Ty::Arr || B.k == Ty::TexArr ? B.n : 0;
        if (!n) invalid(e->line, e->col, "cannot index " + tname(B));
        if (i->has_cv) {
            if (i->cv.iv[0] < 0 || i->cv.iv[0] >= n) invalid(i->line, i->col, "index " + std::to_string(i->cv.iv[0]) + " out of bounds for " + tname(B));
            conv(i, scalar(S_I32));
        }
        std::string ci = code(i);
        if (B.k == Ty::TexArr) {
            e->code = ci;   // only textureSample / textureDimensions take it
            Ty t;
            t.k = Ty::Tex;
            return set(e, t);
        }
        std::string idx = "wg_idx(" + ci + ", " + std::to_string(n) + "u)";
        if (b->uref) {
            uint32_t a, s;
            Ty el = B.k == Ty::Arr ? *B.el : B.k == Ty::Mat ? vec(S_F32, B.m) : scalar(B.s);
            layout(el, a, s, e->line, e->col);
            uint32_t stride = B.k == Ty::Arr ? (s + a - 1) / a * a : B.k == Ty::Mat ? (B.m == 2 ? 8 : 16) : 4;
            e->code = b->code + " + " + std::to_string(stride) + " * " + idx;
            e->uref = true;
            return set(e, el);
        }
        std::string cb = code(b);
        if (B.k == Ty::Vec) { e->code = cb + ".v[" + idx + "]"; return set(e, scalar(B.s)); }
        if (B.k == Ty::Mat) { e->code = cb + ".c[" + idx + "]"; return set(e, vec(S_F32, B.m)); }
        e->code = cb + ".a[" + idx + "]";
        return set(e, *B.el);
    }


    Ty check_member(const ExprP &e) {
        const ExprP &b = e->a[0];
        Ty B = check(b);
        const std::string &mname = e->s;
        if (B.k == Ty::Struct) {
            const StructInfo &si = structs[B.sid];
            for (const FieldInfo &f : si.fields) {
                if (f.name != mname) continue;
                if (b->uref) {
                    e->code = b->code + " + " + std::to_string(f.offset);
                    e->uref = true;
                } else {
                    e->code = code(b) + ".m_" + mname;
                }
                return set(e, f.ty);
            }
            invalid(e->line, e->col, "struct " + si.name + " has no member '" + mname + "'");
        }
        if (B.k == Ty::Vec) {
            std::vector<int> idx;
            bool xyzw = false, rgba = false;
            for (char c : mname) {
                const char *p1 = strchr("xyzw", c), *p2 = strchr("rgba", c);
                if (p1 && c) { idx.push_back((int)(p1 - "xyzw")); xyzw = true; }
                else if (p2 && c) { idx.push_back((int)(p2 - "rgba")); rgba = true; }
                else invalid(e->line, e->col, "invalid swizzle '" + mname + "'");
            }
            if ((xyzw && rgba) || idx.size() > 4) invalid(e->line, e->col, "invalid swizzle '" + mname + "'");
            for (int k : idx) if (k >= B.n) invalid(e->line, e->col, "swizzle '" + mname + "' out of bounds for " + tname(B));
            if (b->has_cv) {
                CV cv;
                cv.f = b->cv.f;
                cv.n = idx.size() == 1 ? 0 : (int)idx.size();
                for (size_t k = 0; k < idx.size(); k++) { cv.fv[k] = b->cv.fv[idx[k]]; cv.iv[k] = b->cv.iv[idx[k]]; }
                return set_cv(e, cv);
            }
            std::string cb = code(b);
            if (idx.size() == 1) { e->code = cb + ".v[" + std::to_string(idx[0]) + "]"; return set(e, scalar(B.s)); }
            std::string s = "wsw<";
            for (size_t k = 0; k < idx.size(); k++) s += (k ? ", " : "") + std::to_string(idx[k]);
            e->code = s + ">(" + cb + ")";
            return set(e, vec(B.s, (int)idx.size()));
        }
        invalid(e->line, e->col, "no member '" + mname + "' on " + tname(B));
    }

    std::string value(const ExprP &e) { return code(e); }

    // f(operands).  WGSL evaluates operands left to right and C++ leaves a call's argument order unspecified; that is
    // only visible once a call can write var<private> state, so in a module with var<private>, operands of which two
    // or more call a user function or read private state are evaluated in order into temporaries first.
    bool has_private = false;
    std::string ordered(const std::string &f, const std::vector<std::string> &ops) {
        int touching = 0;
        bool call = false;
        for (const std::string &o : ops) {
            const bool c = o.find("fn_") != std::string::npos;
            call = call || c;
            touching += c || o.find("ctx.pv.") != std::string::npos;
        }
        std::string s;
        if (!has_private || !call || touching < 2) {
            for (size_t i = 0; i < ops.size(); i++) s += (i ? ", " : "") + ops[i];
            return f + "(" + s + ")";
        }
        std::string args;
        for (size_t i = 0; i < ops.size(); i++) {   // values, copied: a later operand may write what an earlier one read
            const std::string t = ops[i] == "ctx" ? ops[i] : "wg_o" + std::to_string(i);
            if (t != ops[i]) s += "const auto " + t + " = " + ops[i] + "; ";
            args += (i ? ", " : "") + t;
        }
        return "[&]() { " + s + "return " + f + "(" + args + "); }()";
    }

    // the type expression an alias names, followed to a type that is not an alias
    TypeP dealias(TypeP tp) {
        std::set<std::string> seen;
        for (auto it = aliases.find(tp->name); it != aliases.end() && tp->targs.empty(); it = aliases.find(tp->name)) {
            if (!seen.insert(tp->name).second) invalid(it->second->line, it->second->col, "alias " + tp->name + " refers to itself");
            tp = it->second->ty;
        }
        return tp;
    }

    Ty check_call(const ExprP &e) {
        const TypeP c = dealias(e->callee);
        const std::string &n = c->name;
        for (const char *u : kUnsupportedFns) if (n == u) unsupported(e->line, e->col, n);
        std::vector<Ty> A;
        if (!kTextureFns.count(n))
            for (auto &x : e->a) A.push_back(check(x));
        auto args = [&](const std::vector<Ty> &to) {
            std::string s;
            for (size_t i = 0; i < e->a.size(); i++) {
                conv(e->a[i], to[i]);
                s += (i ? ", " : "") + code(e->a[i]);
            }
            return s;
        };
        auto nargs = [&](size_t k) {
            if (e->a.size() != k) invalid(e->line, e->col, n + " expects " + std::to_string(k) + " argument(s), got " + std::to_string(e->a.size()));
        };
        // user functions
        auto uf = fns.find(n);
        if (uf != fns.end()) {
            if (uf->second.d->attrs.size() && (find_attr(uf->second.d->attrs, "vertex") || find_attr(uf->second.d->attrs, "fragment")))
                invalid(e->line, e->col, "an entry point cannot be called");
            nargs(uf->second.params.size());
            if (cur_fn) cur_fn->calls.push_back(n);
            std::vector<std::string> ops = {"ctx"};
            for (size_t i = 0; i < e->a.size(); i++) {
                conv(e->a[i], uf->second.params[i]);
                ops.push_back(code(e->a[i]));
            }
            e->code = ordered(uf->second.cname, ops);
            return set(e, uf->second.ret);
        }
        // structs
        auto st = struct_ids.find(n);
        if (st != struct_ids.end()) {
            resolve_struct(st->second);
            const StructInfo &si = structs[st->second];
            Ty t;
            t.k = Ty::Struct; t.sid = st->second;
            if (e->a.empty()) { e->code = cty(t) + "{}"; return set(e, t); }
            nargs(si.fields.size());
            std::vector<Ty> to;
            for (const FieldInfo &f : si.fields) to.push_back(f.ty);
            e->code = cty(t) + "{" + args(to) + "}";
            return set(e, t);
        }
        // scalar conversions
        if (n == "f32" || n == "i32" || n == "u32" || n == "bool") {
            Ty t = resolve(c);
            if (e->a.empty()) { e->code = cty(t) + "{}"; return set(e, t); }
            nargs(1);
            if (A[0].k != Ty::Scalar) invalid(e->line, e->col, n + "() needs a scalar, found " + tname(A[0]));
            if (e->a[0]->has_cv && t.s != S_BOOL) {   // an abstract argument takes the type (converted, if it is a float)
                const ExprP &x = e->a[0];
                if (x->cv.f && t.s != S_F32) {
                    CV cv;
                    cv.iv[0] = (long long)std::trunc(x->cv.fv[0]);
                    x->cv = cv;
                    x->ty = scalar(S_AI);
                }
                conv(x, t);
                e->code = code(x);
                return set(e, t);
            }
            conv_default(e->a[0]);
            e->code = "wc<" + cty(t) + ">(" + code(e->a[0]) + ")";
            return set(e, t);
        }
        if (n == "bitcast") {
            Ty t = resolve(c->targs.size() == 1 ? c->targs[0] : c);
            nargs(1);
            conv_default(e->a[0]);
            Ty a = e->a[0]->ty;
            if (!(a.k == Ty::Scalar && t.k == Ty::Scalar && a.s != S_BOOL && t.s != S_BOOL))
                unsupported(e->line, e->col, "bitcast other than between 32-bit scalars");
            e->code = "wbits<" + cty(t) + ">(" + code(e->a[0]) + ")";
            return set(e, t);
        }
        // vectors
        bool vecn = n.size() >= 4 && n.compare(0, 3, "vec") == 0 && n[3] >= '2' && n[3] <= '4' && (n.size() == 4 || n.size() == 5);
        if (vecn) {
            int N = n[3] - '0';
            SK s;
            bool inferred = c->targs.empty() && n.size() == 4;
            if (!inferred) s = resolve(c).s;
            else {
                if (e->a.empty()) invalid(e->line, e->col, n + "() without a type needs arguments");
                s = A[0].s;
                for (size_t i = 1; i < A.size(); i++) s = unify(s, A[i].s, e->a[i]);
            }
            if (e->a.empty()) { e->code = cty(vec(s, N)) + "{}"; return set(e, vec(s, N)); }
            if (e->a.size() == 1 && A[0].k == Ty::Scalar) {   // splat
                if (e->a[0]->has_cv && abstract(scalar(s))) {
                    CV cv = e->a[0]->cv;
                    cv.n = N;
                    for (int i = 1; i < N; i++) { cv.fv[i] = cv.fv[0]; cv.iv[i] = cv.iv[0]; }
                    return set_cv(e, cv);
                }
                s = concrete_of(s);
                if (!inferred && !convertible(A[0].s, s)) {
                    conv_default(e->a[0]);
                    e->code = "wsplat<" + std::to_string(N) + ">(wc<" + cscalar(s) + ">(" + code(e->a[0]) + "))";
                } else {
                    conv(e->a[0], scalar(s));
                    e->code = "wsplat<" + std::to_string(N) + ">(" + code(e->a[0]) + ")";
                }
                return set(e, vec(s, N));
            }
            if (e->a.size() == 1 && A[0].k == Ty::Vec && A[0].n == N && !convertible(A[0].s, s)) {   // conversion
                conv_default(e->a[0]);
                e->code = "wc<" + cscalar(s) + ">(" + code(e->a[0]) + ")";
                return set(e, vec(s, N));
            }
            int total = 0;
            bool all_cv = true;
            for (size_t i = 0; i < A.size(); i++) {
                if (A[i].k == Ty::Scalar) total += 1;
                else if (A[i].k == Ty::Vec) total += A[i].n;
                else invalid(e->a[i]->line, e->a[i]->col, "a vector component cannot be " + tname(A[i]));
                all_cv = all_cv && e->a[i]->has_cv;
            }
            if (total != N) invalid(e->line, e->col, n + " needs " + std::to_string(N) + " components, got " + std::to_string(total));
            if (all_cv && abstract(scalar(s))) {
                CV cv;
                cv.f = s == S_AF;
                cv.n = N;
                int k = 0;
                for (auto &x : e->a)
                    for (int j = 0; j < std::max(1, x->cv.n); j++, k++) {
                        cv.fv[k] = x->cv.f ? x->cv.fv[j] : (double)x->cv.iv[j];
                        cv.iv[k] = x->cv.iv[j];
                    }
                return set_cv(e, cv);
            }
            s = concrete_of(s);
            std::vector<std::string> parts;
            for (size_t i = 0; i < A.size(); i++) {
                conv(e->a[i], with_elem(A[i], s));
                parts.push_back(code(e->a[i]));
            }
            e->code = ordered("wvec<" + cscalar(s) + ", " + std::to_string(N) + ">", parts);
            return set(e, vec(s, N));
        }
        if (n.compare(0, 3, "mat") == 0 && (n.size() == 6 || n.size() == 7) && n[4] == 'x') {
            Ty t;
            if (c->targs.empty() && n.size() == 6) { t.k = Ty::Mat; t.n = n[3] - '0'; t.m = n[5] - '0'; }
            else t = resolve(c);
            if (t.k != Ty::Mat || t.n < 2 || t.n > 4 || t.m < 2 || t.m > 4) invalid(e->line, e->col, "unknown type " + n);
            if (e->a.empty()) { e->code = cty(t) + "{}"; return set(e, t); }
            if (e->a.size() == 1 && A[0] == t) { e->code = code(e->a[0]); return set(e, t); }
            int total = 0;
            std::vector<std::string> parts;
            for (size_t i = 0; i < A.size(); i++) {
                if (A[i].k == Ty::Scalar) total += 1;
                else if (A[i].k == Ty::Vec && A[i].n == t.m) total += t.m;
                else invalid(e->a[i]->line, e->a[i]->col, "a matrix constructor takes scalars or column vectors");
                conv(e->a[i], with_elem(A[i], S_F32));
                parts.push_back(code(e->a[i]));
            }
            if (total != t.n * t.m) invalid(e->line, e->col, n + " needs " + std::to_string(t.n * t.m) + " components");
            e->code = ordered("wmat<" + std::to_string(t.n) + ", " + std::to_string(t.m) + ">", parts);
            return set(e, t);
        }
        if (n == "array") {
            Ty t;
            if (c->targs.empty()) {
                if (e->a.empty()) invalid(e->line, e->col, "array() without a type needs arguments");
                Ty el = A[0];
                for (size_t i = 1; i < A.size(); i++) {
                    if (abstract(el) && A[i] != el && (A[i].k == el.k && A[i].n == el.n)) el = with_elem(el, unify(el.s, A[i].s, e->a[i]));
                }
                t.k = Ty::Arr; t.el = std::make_shared<Ty>(concrete(el)); t.n = (int)A.size();
            } else {
                t = resolve(c);
            }
            if (e->a.empty()) { e->code = cty(t) + "{}"; return set(e, t); }
            nargs((size_t)t.n);
            std::vector<Ty> to(e->a.size(), *t.el);
            e->code = cty(t) + "{{" + args(to) + "}}";
            return set(e, t);
        }
        // texture builtins: a texture value (textures[i], or a let or parameter holding one) and the sampler
        auto tex_arg = [&](size_t i) {
            Ty tt = check(e->a[i]);
            if (tt.k != Ty::Tex) invalid(e->line, e->col, n + " takes a texture_2d<f32>, such as textures[i]");
            return "(unsigned)(" + e->a[i]->code + ")";
        };
        auto samp_arg = [&](size_t i) {
            if (check(e->a[i]).k != Ty::Samp) invalid(e->line, e->col, n + " takes the sampler");
        };
        auto val_arg = [&](size_t i, const Ty &t) {
            check(e->a[i]);
            conv(e->a[i], t);
            return code(e->a[i]);
        };
        if (n == "textureSample") {
            nargs(3);
            std::string t = tex_arg(0);
            samp_arg(1);
            e->code = ordered("ctx.tex.sample", {t, val_arg(2, vec(S_F32, 2))});
            return set(e, vec(S_F32, 4));
        }
        if (n == "textureSampleLevel" || n == "textureSampleBias" || n == "textureSampleGrad" || n == "textureSampleBaseClampToEdge" ||
            n == "textureGather") {
            const bool gather = n == "textureGather";
            const size_t k = n == "textureSampleGrad" ? 5 : n == "textureSampleBaseClampToEdge" ? 3 : 4;
            if (e->a.size() == k + 1 && n != "textureSampleBaseClampToEdge") unsupported(e->line, e->col, n + " with an offset");
            nargs(k);
            std::vector<std::string> ops;
            if (gather) {   // textureGather(component, t, s, coords): the component is a const-expression in 0..3
                const ExprP &c = e->a[0];
                Ty ct = check(c);
                if (ct.k != Ty::Scalar || !integral(ct.s)) invalid(c->line, c->col, "textureGather's component must be i32 or u32, found " + tname(ct));
                long long v;
                if (c->has_cv && !c->cv.f && !c->cv.n) v = c->cv.iv[0];
                else if (c->cint) v = c->civ;
                else invalid(c->line, c->col, "textureGather's component must be a const-expression");
                if (v < 0 || v > 3) invalid(c->line, c->col, "textureGather's component must be 0, 1, 2 or 3, found " + std::to_string(v));
                ops.push_back(std::to_string(v));
            }
            const size_t o = gather ? 1 : 0;
            ops.push_back(tex_arg(o));
            samp_arg(o + 1);
            ops.push_back(val_arg(o + 2, vec(S_F32, 2)));
            if (n == "textureSampleBias" && cur_fn && !cur_fn->frag_line) { cur_fn->frag_line = e->line; cur_fn->frag_col = e->col; }
            if (n == "textureSampleLevel" || n == "textureSampleBias") ops.push_back(val_arg(3, scalar(S_F32)));
            if (n == "textureSampleGrad") { ops.push_back(val_arg(3, vec(S_F32, 2))); ops.push_back(val_arg(4, vec(S_F32, 2))); }
            const char *m = n == "textureSampleLevel" ? "sample_level" : n == "textureSampleBias" ? "sample_bias" :
                            n == "textureSampleGrad" ? "sample_grad" : gather ? "gather" : "sample_clamped";
            e->code = ordered(std::string("ctx.tex.") + m, ops);
            return set(e, vec(S_F32, 4));
        }
        if (n == "textureDimensions" || n == "textureNumLevels") {
            const bool dims = n == "textureDimensions";
            if (e->a.size() != 1 && !(dims && e->a.size() == 2)) nargs(1);
            std::string t = tex_arg(0);
            if (!dims) {
                e->code = "ctx.tex.levels(" + t + ")";
                return set(e, scalar(S_U32));
            }
            if (e->a.size() == 2) {   // any level: a node texture's size (levels are clamped to its one level)
                Ty l = check(e->a[1]);
                if (l.k != Ty::Scalar || !integral(l.s)) invalid(e->a[1]->line, e->a[1]->col, "textureDimensions' level must be i32 or u32, found " + tname(l));
                conv_default(e->a[1]);
                e->code = ordered("ctx.tex.dims", {t, code(e->a[1])});
                return set(e, vec(S_U32, 2));
            }
            e->code = "ctx.tex.dims(" + t + ")";
            return set(e, vec(S_U32, 2));
        }
        // math builtins
        static const std::set<std::string> f1 = {"floor", "ceil", "fract", "round", "trunc", "sqrt", "inverseSqrt", "exp", "exp2",
                                                 "log", "log2", "sin", "cos", "tan", "asin", "acos", "atan", "saturate",
                                                 "degrees", "radians", "sinh", "cosh", "tanh", "asinh", "acosh", "atanh",
                                                 "quantizeToF16"};
        auto fv = [&](const Ty &t) { return (t.k == Ty::Scalar || t.k == Ty::Vec) && (t.s == S_F32 || t.s == S_AF || t.s == S_AI); };
        auto common = [&](bool floats) {   // every argument to one type (scalars and vectors as they are)
            SK s = A[0].s;
            for (size_t i = 1; i < A.size(); i++) s = unify(s, A[i].s, e->a[i]);
            s = floats && s == S_AI ? S_F32 : concrete_of(s);
            return s;
        };
        auto fin = [&](const Ty &r) {
            std::vector<std::string> ops;
            for (size_t i = 0; i < e->a.size(); i++) ops.push_back(code(e->a[i]));
            e->code = ordered("wb_" + n, ops);
            return set(e, r);
        };
        if (f1.count(n)) {
            nargs(1);
            if (!fv(A[0])) invalid(e->line, e->col, n + " needs f32 or vecN<f32>, found " + tname(A[0]));
            conv(e->a[0], with_elem(A[0], S_F32));
            return fin(with_elem(A[0], S_F32));
        }
        if (n == "abs" || n == "sign") {
            nargs(1);
            if (!(A[0].k == Ty::Scalar || A[0].k == Ty::Vec) || !numeric(A[0].s) || (n == "sign" && A[0].s == S_U32))
                invalid(e->line, e->col, n + " needs a number, found " + tname(A[0]));
            conv_default(e->a[0]);
            return fin(concrete(A[0]));
        }
        if (n == "min" || n == "max" || n == "clamp" || n == "atan2" || n == "pow" || n == "step" || n == "mix" || n == "smoothstep" ||
            n == "fma") {
            size_t k = n == "clamp" || n == "mix" || n == "smoothstep" || n == "fma" ? 3 : 2;
            nargs(k);
            bool floats = !(n == "min" || n == "max" || n == "clamp");
            for (const Ty &t : A)
                if (!(t.k == Ty::Scalar || t.k == Ty::Vec) || !numeric(t.s) || (floats && !fv(t))) invalid(e->line, e->col, n + " does not take " + tname(t));
            SK s = common(floats);
            Ty shape = A[0].k == Ty::Vec ? A[0] : A.back();
            for (const Ty &t : A) if (t.k == Ty::Vec) shape = t;
            Ty r = with_elem(shape, s);
            std::vector<std::string> parts;
            for (size_t i = 0; i < k; i++) {
                bool scalar_ok = n == "mix" && i == 2;   // mix(vec, vec, f32)
                if (A[i].k != r.k || A[i].n != r.n) {
                    if (!(scalar_ok && A[i].k == Ty::Scalar)) invalid(e->a[i]->line, e->a[i]->col, n + ": mismatched argument " + tname(A[i]));
                    conv(e->a[i], scalar(s));
                    parts.push_back("wsplat<" + std::to_string(r.n) + ">(" + code(e->a[i]) + ")");
                } else {
                    conv(e->a[i], r);
                    parts.push_back(code(e->a[i]));
                }
            }
            e->code = ordered("wb_" + n, parts);
            return set(e, r);
        }
        if (n == "length" || n == "normalize" || n == "dot" || n == "distance" || n == "cross") {
            size_t k = n == "length" || n == "normalize" ? 1 : 2;
            nargs(k);
            SK s = common(n != "dot");
            for (size_t i = 0; i < k; i++) {
                if (A[i].k != A[0].k || A[i].n != A[0].n) invalid(e->line, e->col, n + ": mismatched arguments");
                conv(e->a[i], with_elem(A[i], s));
            }
            if (n == "dot" && (A[0].k != Ty::Vec || s == S_BOOL)) invalid(e->line, e->col, "dot needs vectors");
            if ((n == "normalize") && A[0].k != Ty::Vec) invalid(e->line, e->col, "normalize needs a vector");
            if (n == "cross" && (A[0].k != Ty::Vec || A[0].n != 3 || s != S_F32)) invalid(e->line, e->col, "cross needs vec3<f32>");
            if (n != "dot" && s != S_F32) invalid(e->line, e->col, n + " needs f32");
            Ty r = n == "normalize" || n == "cross" ? vec(s, A[0].n) : scalar(s);
            return fin(r);
        }
        if (n == "select") {
            nargs(3);
            Ty C = A[2];
            if (!((C.k == Ty::Scalar || C.k == Ty::Vec) && C.s == S_BOOL)) invalid(e->line, e->col, "select's condition must be bool");
            if (A[0].k != A[1].k || A[0].n != A[1].n) invalid(e->line, e->col, "select: mismatched arguments");
            if (C.k == Ty::Vec && (A[0].k != Ty::Vec || A[0].n != C.n)) invalid(e->line, e->col, "select: condition size mismatch");
            Ty r = A[0];
            if (abstract(A[0]) || abstract(A[1])) r = concrete(with_elem(A[0], unify(A[0].s, A[1].s, e)));
            conv(e->a[0], r); conv(e->a[1], r);
            return fin(r);
        }
        if (n == "any" || n == "all") {
            nargs(1);
            if (A[0].s != S_BOOL) invalid(e->line, e->col, n + " needs bool");
            return fin(scalar(S_BOOL));
        }
        if (n == "transpose") {
            nargs(1);
            if (A[0].k != Ty::Mat) invalid(e->line, e->col, "transpose needs a matrix");
            Ty r = A[0];
            std::swap(r.n, r.m);
            return fin(r);
        }
        if (n == "ldexp") {
            nargs(2);
            if (!fv(A[0])) invalid(e->line, e->col, "ldexp needs f32 or vecN<f32>, found " + tname(A[0]));
            if (A[1].k != A[0].k || A[1].n != A[0].n || !(A[1].s == S_I32 || A[1].s == S_AI))
                invalid(e->a[1]->line, e->a[1]->col, "ldexp's exponent must be " + tname(with_elem(A[0], S_I32)) + ", found " + tname(A[1]));
            conv(e->a[0], with_elem(A[0], S_F32));
            conv(e->a[1], with_elem(A[1], S_I32));
            return fin(with_elem(A[0], S_F32));
        }
        if (n == "frexp" || n == "modf") {
            nargs(1);
            if (!fv(A[0])) invalid(e->line, e->col, n + " needs f32 or vecN<f32>, found " + tname(A[0]));
            Ty f = with_elem(A[0], S_F32);
            conv(e->a[0], f);
            return fin(result_struct(n, f));
        }
        if (n == "determinant") {
            nargs(1);
            if (A[0].k != Ty::Mat || A[0].n != A[0].m) invalid(e->line, e->col, "determinant needs a square matrix, found " + tname(A[0]));
            return fin(scalar(S_F32));
        }
        if (n == "faceForward" || n == "reflect" || n == "refract") {
            const size_t k = n == "reflect" ? 2 : 3, nv = n == "refract" ? 2 : k;
            nargs(k);
            if (A[0].k != Ty::Vec || !fv(A[0])) invalid(e->line, e->col, n + " needs vecN<f32>, found " + tname(A[0]));
            const Ty v = with_elem(A[0], S_F32);
            for (size_t i = 0; i < k; i++) {
                const Ty want = i < nv ? v : scalar(S_F32);
                if (A[i].k != want.k || A[i].n != want.n || !fv(A[i])) invalid(e->a[i]->line, e->a[i]->col, n + ": expected " + tname(want) + ", found " + tname(A[i]));
                conv(e->a[i], want);
            }
            return fin(v);
        }
        // bit builtins: i32, u32 and vectors of them
        auto iv = [&](const Ty &t) { return (t.k == Ty::Scalar || t.k == Ty::Vec) && (t.s == S_I32 || t.s == S_U32 || t.s == S_AI); };
        static const std::set<std::string> b1 = {"countOneBits", "countLeadingZeros", "countTrailingZeros", "reverseBits",
                                                 "firstTrailingBit", "firstLeadingBit"};
        if (b1.count(n) || n == "extractBits" || n == "insertBits") {
            const size_t k = b1.count(n) ? 1 : n == "extractBits" ? 3 : 4, nv = n == "insertBits" ? 2 : 1;
            nargs(k);
            if (!iv(A[0])) invalid(e->line, e->col, n + " needs i32, u32 or a vector of them, found " + tname(A[0]));
            Ty t = concrete(A[0]);
            if (nv == 2) {
                if (!iv(A[1]) || A[1].k != A[0].k || A[1].n != A[0].n) invalid(e->a[1]->line, e->a[1]->col, n + ": mismatched argument " + tname(A[1]));
                t = concrete(with_elem(A[0], unify(A[0].s, A[1].s, e)));
            }
            for (size_t i = 0; i < k; i++) {
                if (i < nv) { conv(e->a[i], t); continue; }
                if (A[i].k != Ty::Scalar || !(A[i].s == S_U32 || A[i].s == S_AI))
                    invalid(e->a[i]->line, e->a[i]->col, n + "'s offset and count must be u32, found " + tname(A[i]));
                conv(e->a[i], scalar(S_U32));
            }
            return fin(t);
        }
        if (n == "dot4U8Packed" || n == "dot4I8Packed") {
            nargs(2);
            for (size_t i = 0; i < 2; i++) {
                if (A[i].k != Ty::Scalar || !(A[i].s == S_U32 || A[i].s == S_AI)) invalid(e->a[i]->line, e->a[i]->col, n + " needs u32, found " + tname(A[i]));
                conv(e->a[i], scalar(S_U32));
            }
            return fin(scalar(n == "dot4U8Packed" ? S_U32 : S_I32));
        }
        // packing: pack4x8* / pack2x16* take vec4 / vec2<f32>, unpack* give them
        if (n.compare(0, 4, "pack") == 0 && (n == "pack4x8snorm" || n == "pack4x8unorm" || n == "pack2x16snorm" ||
                                             n == "pack2x16unorm" || n == "pack2x16float")) {
            nargs(1);
            const int N = n[4] == '4' ? 4 : 2;
            if (A[0].k != Ty::Vec || A[0].n != N || !fv(A[0])) invalid(e->line, e->col, n + " needs " + tname(vec(S_F32, N)) + ", found " + tname(A[0]));
            conv(e->a[0], vec(S_F32, N));
            return fin(scalar(S_U32));
        }
        if (n == "unpack4x8snorm" || n == "unpack4x8unorm" || n == "unpack2x16snorm" || n == "unpack2x16unorm" || n == "unpack2x16float") {
            nargs(1);
            if (A[0].k != Ty::Scalar || !(A[0].s == S_U32 || A[0].s == S_AI)) invalid(e->line, e->col, n + " needs u32, found " + tname(A[0]));
            conv(e->a[0], scalar(S_U32));
            return fin(vec(S_F32, n[6] == '4' ? 4 : 2));
        }
        invalid(e->line, e->col, "unknown function '" + n + "'");
    }

    // the predeclared result struct of frexp / modf for f32 or vecN<f32>: __frexp_result_f32 { fract, exp },
    // __modf_result_vec2_f32 { fract, whole }, ...
    std::map<std::string, int> result_structs;
    Ty result_struct(const std::string &fn, const Ty &f) {
        const std::string name = "__" + fn + "_result_" + (f.k == Ty::Vec ? "vec" + std::to_string(f.n) + "_" : "") + "f32";
        auto it = result_structs.find(name);
        Ty t;
        t.k = Ty::Struct;
        if (it != result_structs.end()) { t.sid = it->second; return t; }
        StructInfo si;
        si.name = name;
        si.resolved = true;
        const Ty second = fn == "frexp" ? with_elem(f, S_I32) : f;
        si.fields = {FieldInfo{"fract", f, {}, 0}, FieldInfo{fn == "frexp" ? "exp" : "whole", second, {}, 0}};
        si.cname = fn == "frexp" ? "wfrexp<" + cty(f) + ", " + cty(second) + ">" : "wmodf<" + cty(f) + ">";
        t.sid = (int)structs.size();
        structs.push_back(si);
        result_structs[name] = t.sid;
        return t;
    }

    // ---- const-expressions: const_assert evaluates them here, with WGSL's rules for const-expressions ----
    // Concrete f32 results are rounded to f32 after each operation; abstract ones stay f64 / int64, and a comparison of two
    // abstract operands compares them unconverted.  Overflow, a non-finite float, division by zero and a shift by the bit
    // width or more are errors, as WGSL makes them for const-expressions.
    [[noreturn]] void not_const(const ExprP &e) { invalid(e->line, e->col, "not a const-expression"); }
    static bool is_float(SK s) { return s == S_F32 || s == S_AF; }

    double kv_float(const KV &v, int k, int line, int col, SK to) {
        double d = is_float(v.s) ? v.f[k] : (double)v.i[k];
        if (to == S_F32) d = (float)d;
        if (!std::isfinite(d)) invalid(line, col, "constant expression overflows");
        return d;
    }
    long long kv_int(long double x, SK to, int line, int col) {
        const long double lo = to == S_I32 ? -2147483648.0L : to == S_U32 ? 0.0L : -9223372036854775808.0L;
        const long double hi = to == S_I32 ? 2147483647.0L : to == S_U32 ? 4294967295.0L : 9223372036854775807.0L;
        if (!(x >= lo && x <= hi)) invalid(line, col, "constant expression overflows " + sname(to));
        return (long long)x;
    }
    // a component converted to `to` as a value constructor converts it (f32 -> integer truncates and saturates)
    KV kv_convert(const KV &v, SK to, int line, int col) {
        KV r = v;
        r.s = to;
        for (int k = 0; k < std::max(1, v.n); k++) {
            if (is_float(to)) { r.f[k] = kv_float(v, k, line, col, to); continue; }
            if (to == S_BOOL) { r.i[k] = is_float(v.s) ? v.f[k] != 0.0 : v.i[k] != 0; continue; }
            if (!is_float(v.s)) {   // i32 <-> u32 keep the bits
                r.i[k] = to == S_U32 ? (long long)(uint32_t)v.i[k] : to == S_I32 ? (long long)(int32_t)(uint32_t)v.i[k] : v.i[k];
                continue;
            }
            const double x = std::trunc(v.f[k]);
            r.i[k] = x != x ? 0 : to == S_U32 ? (x < 0 ? 0 : x > 4294967295.0 ? 4294967295LL : (long long)x)
                                              : (x < -2147483648.0 ? -2147483648LL : x > 2147483647.0 ? 2147483647LL : (long long)x);
        }
        return r;
    }

    KV ceval(const ExprP &e, bool keep_abstract = false) {
        if (e->has_cv) {
            KV r;
            r.s = e->cv.f ? S_AF : S_AI;
            r.n = e->cv.n;
            for (int k = 0; k < 4; k++) { r.f[k] = e->cv.fv[k]; r.i[k] = e->cv.iv[k]; }
            if (keep_abstract) return r;
            const SK to = e->has_target ? e->target.s : concrete_of(r.s);
            if (!is_float(to)) for (int k = 0; k < std::max(1, r.n); k++) lit(e->cv, k, to, e->line, e->col);   // range
            return kv_convert(r, to, e->line, e->col);
        }
        const Ty &t = e->ty;
        KV r;
        r.s = t.s;
        r.n = t.k == Ty::Vec ? t.n : 0;
        const bool value_type = t.k == Ty::Scalar || t.k == Ty::Vec;
        switch (e->k) {
            case Expr::Lit:
                if (e->lk == 'b') r.i[0] = e->bv;
                else if (r.s == S_F32) r.f[0] = (float)e->fv;
                else r.i[0] = e->iv;
                return r;
            case Expr::Id: {
                Sym *s = lookup(e->s);
                if (!s || !s->is_const) not_const(e);
                if (s->kv_status == SMR_ERR_UNSUPPORTED) unsupported(e->line, e->col, "const_assert over '" + e->s + "', which is not evaluated at translation");
                if (s->kv_status) invalid(e->line, e->col, "'" + e->s + "' is not a const-expression");
                return s->kv;
            }
            case Expr::Un: {
                const KV a = ceval(e->a[0]);
                for (int k = 0; k < std::max(1, r.n); k++) {
                    if (e->s == "!") r.i[k] = !a.i[k];
                    else if (e->s == "~") r.i[k] = r.s == S_U32 ? (long long)(uint32_t)~a.i[k] : ~a.i[k];
                    else if (is_float(r.s)) r.f[k] = -a.f[k];
                    else r.i[k] = kv_int(-(long double)a.i[k], r.s, e->line, e->col);
                }
                return r;
            }
            case Expr::Bin: return ceval_binary(e, r);
            case Expr::Idx: {
                const KV b = ceval(e->a[0]), i = ceval(e->a[1]);
                if (!value_type || !b.n) unsupported(e->line, e->col, "const_assert over elements of " + tname(e->a[0]->ty));
                if (i.i[0] < 0 || i.i[0] >= b.n) invalid(e->a[1]->line, e->a[1]->col, "index out of bounds");
                r = b;
                r.n = 0;
                r.f[0] = b.f[i.i[0]]; r.i[0] = b.i[i.i[0]];
                return r;
            }
            case Expr::Mem: {
                const KV b = ceval(e->a[0]);
                if (e->a[0]->ty.k != Ty::Vec) unsupported(e->line, e->col, "const_assert over struct members");
                for (size_t k = 0; k < e->s.size(); k++) {
                    const char *c = strchr("xyzw", e->s[k]);
                    const int j = c ? (int)(c - "xyzw") : (int)(strchr("rgba", e->s[k]) - "rgba");
                    r.f[k] = b.f[j]; r.i[k] = b.i[j];
                }
                return r;
            }
            case Expr::Call: {
                const TypeP c = dealias(e->callee);
                const std::string &n = c->name;
                if (fns.count(n) || kTextureFns.count(n)) not_const(e);
                std::vector<KV> A;
                for (const ExprP &x : e->a) A.push_back(ceval(x));
                if (!value_type) unsupported(e->line, e->col, "const_assert over " + tname(t) + " values");
                if (A.empty()) return r;   // the zero value
                if (n == "f32" || n == "i32" || n == "u32" || n == "bool" || (t.k == Ty::Vec && A.size() == 1 && A[0].n == r.n))
                    return kv_convert(A[0], r.s, e->line, e->col);
                if (t.k == Ty::Vec && n.compare(0, 3, "vec") == 0) {   // components in order, or one scalar splatted
                    int k = 0;
                    for (const KV &a : A) {
                        const KV v = kv_convert(a, r.s, e->line, e->col);
                        for (int j = 0; j < std::max(1, a.n); j++, k++) { r.f[k] = v.f[j]; r.i[k] = v.i[j]; }
                    }
                    for (; k < r.n; k++) { r.f[k] = r.f[0]; r.i[k] = r.i[0]; }
                    return r;
                }
                if ((n == "all" || n == "any") && A.size() == 1) {
                    bool all = true, any = false;
                    for (int k = 0; k < std::max(1, A[0].n); k++) { all = all && A[0].i[k]; any = any || A[0].i[k]; }
                    r.i[0] = n == "all" ? all : any;
                    return r;
                }
                if (n == "select" && A.size() == 3) {
                    const KV f = kv_convert(A[0], r.s, e->line, e->col), tr = kv_convert(A[1], r.s, e->line, e->col);
                    for (int k = 0; k < std::max(1, r.n); k++) {
                        const bool c2 = A[2].i[A[2].n ? k : 0] != 0;
                        r.f[k] = c2 ? tr.f[k] : f.f[k]; r.i[k] = c2 ? tr.i[k] : f.i[k];
                    }
                    return r;
                }
                if ((n == "abs" || n == "min" || n == "max") && A.size() == (n == "abs" ? 1u : 2u)) {
                    for (int k = 0; k < std::max(1, r.n); k++) {
                        const KV x = kv_convert(A[0], r.s, e->line, e->col), y = kv_convert(A.back(), r.s, e->line, e->col);
                        const int ka = A[0].n ? k : 0, kb = A.back().n ? k : 0;
                        if (is_float(r.s)) r.f[k] = n == "abs" ? std::fabs(x.f[ka]) : n == "min" ? std::fmin(x.f[ka], y.f[kb]) : std::fmax(x.f[ka], y.f[kb]);
                        else r.i[k] = n == "abs" ? (r.s == S_I32 ? (long long)(int32_t)(uint32_t)std::llabs(x.i[ka]) : std::llabs(x.i[ka]))
                                                 : n == "min" ? std::min(x.i[ka], y.i[kb]) : std::max(x.i[ka], y.i[kb]);
                    }
                    return r;
                }
                unsupported(e->line, e->col, n + " in a const_assert");
            }
        }
        return r;
    }

    KV ceval_binary(const ExprP &e, KV r) {
        const std::string &op = e->s;
        const bool cmp = op == "==" || op == "!=" || op == "<" || op == "<=" || op == ">" || op == ">=";
        const bool abs_cmp = cmp && e->a[0]->has_cv && e->a[1]->has_cv;   // two abstract operands compare as they are
        const KV a = ceval(e->a[0], abs_cmp), b = ceval(e->a[1], abs_cmp);
        const int line = e->line, col = e->col;
        if (op == "&&" || op == "||") { r.i[0] = op == "&&" ? (a.i[0] && b.i[0]) : (a.i[0] || b.i[0]); return r; }
        const SK s = a.s;   // the operands' common kind (a shift's count is u32)
        for (int k = 0; k < std::max(1, std::max(a.n, b.n)); k++) {
            const int ka = a.n ? k : 0, kb = b.n ? k : 0;
            if (cmp) {
                int c;
                if (is_float(s) || is_float(b.s)) {
                    const double x = kv_float(a, ka, line, col, S_AF), y = kv_float(b, kb, line, col, S_AF);
                    c = x < y ? -1 : x > y ? 1 : 0;
                } else {
                    c = a.i[ka] < b.i[kb] ? -1 : a.i[ka] > b.i[kb] ? 1 : 0;
                }
                r.i[k] = op == "==" ? c == 0 : op == "!=" ? c != 0 : op == "<" ? c < 0 : op == "<=" ? c <= 0 : op == ">" ? c > 0 : c >= 0;
                continue;
            }
            if (is_float(s)) {
                const double x = a.f[ka], y = b.f[kb];
                auto rd = [&](double v) { return s == S_F32 ? (double)(float)v : v; };
                double v;
                if (op == "+") v = rd(x + y);
                else if (op == "-") v = rd(x - y);
                else if (op == "*") v = rd(x * y);
                else if (op == "/") v = rd(x / y);
                else if (op == "%") v = rd(x - rd(y * std::trunc(rd(x / y))));
                else unsupported(line, col, "'" + op + "' in a const_assert");
                if (!std::isfinite(v)) invalid(line, col, "constant expression overflows");
                r.f[k] = v;
                continue;
            }
            const long long x = a.i[ka], y = b.i[kb];
            if (s == S_BOOL) { r.i[k] = op == "&" ? (x && y) : (x || y); continue; }
            if (op == "&" || op == "|" || op == "^") { r.i[k] = op == "&" ? x & y : op == "|" ? x | y : x ^ y; continue; }
            if (op == "<<" || op == ">>") {
                const int bits = s == S_AI ? 64 : 32;
                if (y < 0 || y >= bits) invalid(line, col, "shift by " + std::to_string(y) + " in a const-expression");
                if (op == ">>") { r.i[k] = s == S_U32 ? (long long)((uint64_t)x >> y) : x >> y; continue; }
                r.i[k] = kv_int((long double)x * std::ldexp(1.0L, (int)y), s, line, col);
                continue;
            }
            if ((op == "/" || op == "%") && y == 0) invalid(line, col, "integer division by zero in a constant expression");
            long double v;   // in long double, where no int64 operation here overflows; kv_int checks the range
            if (op == "+") v = (long double)x + y;
            else if (op == "-") v = (long double)x - y;
            else if (op == "*") v = (long double)x * y;
            else if (op == "/") v = y == -1 ? -(long double)x : (long double)(x / y);
            else v = y == -1 ? 0 : (long double)(x % y);
            r.i[k] = kv_int(v, s, line, col);
        }
        return r;
    }

    // a const declaration's value, for const_assert: evaluated now, or the reason it cannot be
    void const_value(Sym &sym, const ExprP &init) {
        sym.is_const = true;
        if (sym.has_cv) return;   // an abstract constant: its uses carry the value
        try {
            sym.kv = ceval(init);
        } catch (const Fail &f) {
            sym.kv_status = f.status;
        }
    }

    void const_assert(const StmtP &s) {
        const Ty t = check(s->e);
        if (t != scalar(S_BOOL)) invalid(s->e->line, s->e->col, "const_assert needs a bool, found " + tname(t));
        if (!ceval(s->e).i[0]) invalid(s->line, s->col, "const_assert failed");
    }

    // ---- statements ----
    std::string ind(int d) { return std::string(4 * d, ' '); }

    // a reference: a var, or a member / element / component of one
    void check_ref(const ExprP &e) {
        ExprP r = e;
        while (r->k == Expr::Mem || r->k == Expr::Idx) {
            if (r->k == Expr::Mem && r->a[0]->ty.k == Ty::Vec && r->s.size() > 1) invalid(r->line, r->col, "cannot assign to a multi-component swizzle");
            r = r->a[0];
        }
        if (r->k != Expr::Id) invalid(e->line, e->col, "cannot assign to this expression");
        Sym *s = lookup(r->s);
        if (!s || !s->mut) invalid(e->line, e->col, "cannot assign to '" + r->s + "'");
    }

    void push() { scopes.emplace_back(); }
    void pop() { scopes.pop_back(); }
    void declare(const std::string &n, const Sym &s, int line, int col) {
        if (scopes.back().count(n)) invalid(line, col, "redeclaration of '" + n + "'");
        scopes.back()[n] = s;
    }

    void stmts(const std::vector<StmtP> &b, std::string &o, int d) {
        for (const StmtP &s : b) stmt(s, o, d);
    }

    std::string block(const std::vector<StmtP> &b, int d) {
        std::string o = "{\n";
        push();
        stmts(b, o, d + 1);
        pop();
        return o + ind(d) + "}";
    }

    // a texture or sampler is a value a let or a parameter may hold, never a var's or a const's
    void handle_decl(const StmtP &s, const Ty &t) {
        if (t.k == Ty::TexArr) unsupported(s->line, s->col, "binding arrays in local values");
        if ((t.k == Ty::Tex || t.k == Ty::Samp) && s->k != Stmt::Let)
            invalid(s->line, s->col, std::string("a ") + (s->k == Stmt::Var ? "var" : "const") + " cannot hold " + tname(t));
    }

    Ty decl_type(const StmtP &s) {
        Ty t = check(s->e);
        if (t.k == Ty::Void) invalid(s->e->line, s->e->col, "a function without a return value has no value");
        handle_decl(s, t);
        if (s->ty) {
            Ty d = resolve(s->ty);
            handle_decl(s, d);
            conv(s->e, d);
            return d;
        }
        if (s->k != Stmt::Const) { conv_default(s->e); return concrete(t); }
        return t;
    }

    void stmt(const StmtP &s, std::string &o, int d) {
        switch (s->k) {
            case Stmt::Block:
                if (s->body.empty()) return;
                o += ind(d) + block(s->body, d) + "\n";
                return;
            case Stmt::Var: {
                Ty t;
                std::string init;
                if (s->e) { t = decl_type(s); init = value(s->e); }
                else if (s->ty) { t = resolve(s->ty); handle_decl(s, t); }
                else invalid(s->line, s->col, "a var needs a type or an initializer");
                Sym sym;
                sym.k = Sym::Local; sym.ty = t; sym.mut = true; sym.code = "u_" + s->name;
                o += ind(d) + cty(t) + " u_" + s->name + (s->e ? " = " + init : std::string("{}")) + ";\n";
                declare(s->name, sym, s->line, s->col);
                return;
            }
            case Stmt::Let:
            case Stmt::Const: {
                Ty t = decl_type(s);
                Sym sym;
                sym.k = Sym::Local; sym.ty = t;
                if (s->k == Stmt::Const && s->e->has_cv && !s->ty) {
                    sym.has_cv = true; sym.cv = s->e->cv;
                } else {
                    sym.code = "u_" + s->name;
                    if (s->k == Stmt::Const) const_int(sym, s->e);
                    o += ind(d) + "const " + cty(t) + " u_" + s->name + " = " + value(s->e) + ";\n";
                }
                if (s->k == Stmt::Const) const_value(sym, s->e);
                declare(s->name, sym, s->line, s->col);
                return;
            }
            case Stmt::ConstAssert:
                const_assert(s);
                return;
            case Stmt::Phony:
                check(s->e);
                conv_default(s->e);
                o += ind(d) + "(void)(" + value(s->e) + ");\n";
                return;
            case Stmt::Assign: {
                Ty L = check(s->lhs);
                check_ref(s->lhs);
                check(s->e);
                if (s->op == "=") {
                    conv(s->e, L);
                    if (has_private)   // WGSL evaluates the left side first; C++17 evaluates the right operand of = first
                        o += ind(d) + "{ auto &wg_ref_ = " + code(s->lhs) + "; wg_ref_ = " + value(s->e) + "; }\n";
                    else
                        o += ind(d) + code(s->lhs) + " = " + value(s->e) + ";\n";
                    return;
                }
                // e1 op= e2 is e1 = e1 op e2, with e1 evaluated once.  With private state, e1's value is read into wg_val_
                // before e2 is evaluated, as WGSL's `let p = &e1; *p = *p op e2;` does (e2 may call a function writing e1)
                const std::string cur = has_private ? "wg_val_" : "wg_ref_";
                auto bin = std::make_shared<Expr>();
                bin->k = Expr::Bin; bin->line = s->line; bin->col = s->col;
                bin->s = s->op.substr(0, s->op.size() - 1);
                auto ref = std::make_shared<Expr>();
                ref->k = Expr::Id; ref->s = cur; ref->line = s->line; ref->col = s->col;
                push();
                Sym rs;
                rs.ty = L; rs.mut = true; rs.code = cur;
                scopes.back()[cur] = rs;
                bin->a = {ref, s->e};
                s->e->has_target = false;
                Ty r = check(bin);
                pop();
                conv(bin, L);
                if (r != L) invalid(s->line, s->col, "'" + s->op + "' changes the type of the left side");
                o += ind(d) + "{ auto &wg_ref_ = " + code(s->lhs) + "; " + (has_private ? "const auto wg_val_ = wg_ref_; " : "") +
                     "wg_ref_ = " + code(bin) + "; }\n";
                return;
            }
            case Stmt::Incr:
            case Stmt::Decr: {
                Ty L = check(s->lhs);
                check_ref(s->lhs);
                if (L.k != Ty::Scalar || (L.s != S_I32 && L.s != S_U32)) invalid(s->line, s->col, "++ / -- need an i32 or u32 variable");
                std::string one = L.s == S_I32 ? "1" : "1u";
                o += ind(d) + "{ auto &wg_ref_ = " + code(s->lhs) + "; wg_ref_ = " + (s->k == Stmt::Incr ? "w_add" : "w_sub") +
                     "(wg_ref_, " + one + "); }\n";
                return;
            }
            case Stmt::If: {
                Ty c = check(s->e);
                if (c != scalar(S_BOOL)) invalid(s->e->line, s->e->col, "an if condition must be bool, found " + tname(c));
                o += ind(d) + "if (" + code(s->e) + ") " + block(s->body, d);
                if (s->els) {
                    o += " else ";
                    if (s->els->k == Stmt::If) {
                        std::string sub;
                        stmt(s->els, sub, d);
                        o += "{\n" + sub + ind(d) + "}";
                    } else {
                        o += block(s->els->body, d);
                    }
                }
                o += "\n";
                return;
            }
            case Stmt::Switch: {
                Ty t = check(s->e);
                if (t.k != Ty::Scalar || !integral(t.s)) invalid(s->e->line, s->e->col, "a switch selector must be i32 or u32");
                SK sk = t.s;
                for (const Clause &c : s->clauses)
                    for (const ExprP &x : c.sels) {
                        Ty xt = check(x);
                        if (!x->has_cv && !(x->k == Expr::Lit)) invalid(x->line, x->col, "a case selector must be a constant");
                        sk = unify(sk, xt.s, x);
                    }
                sk = concrete_of(sk);
                conv(s->e, scalar(sk));
                o += ind(d) + "switch (" + code(s->e) + ") {\n";
                std::set<long long> seen;
                int defaults = 0;
                loops.push_back(-1);
                for (const Clause &c : s->clauses) {
                    for (const ExprP &x : c.sels) {
                        conv(x, scalar(sk));
                        long long v = x->has_cv ? x->cv.iv[0] : x->iv;   // an abstract constant or a suffixed literal
                        if (!seen.insert(sk == S_U32 ? (long long)(uint32_t)v : v).second) invalid(x->line, x->col, "duplicate case selector");
                        o += ind(d + 1) + "case " + code(x) + ":\n";
                    }
                    if (c.def) { defaults++; o += ind(d + 1) + "default:\n"; }
                    o += ind(d + 1) + block(c.body, d + 1) + "\n" + ind(d + 1) + "break;\n";
                }
                loops.pop_back();
                if (defaults != 1) invalid(s->line, s->col, "a switch needs exactly one default clause");
                o += ind(d) + "}\n";
                return;
            }
            case Stmt::Loop:
            case Stmt::For:
            case Stmt::While: {
                int lab = label++;
                std::string L = "wg_cont_" + std::to_string(lab);
                push();
                std::string pre;
                if (s->k == Stmt::For && s->init) stmt(s->init, pre, d + 1);
                std::string cond;
                if (s->e) {
                    Ty c = check(s->e);
                    if (c != scalar(S_BOOL)) invalid(s->e->line, s->e->col, "a loop condition must be bool, found " + tname(c));
                    cond = code(s->e);
                }
                loops.push_back(lab);
                std::string body = block(s->body, d + 1);
                loops.pop_back();
                std::string cont;
                if (s->k == Stmt::For && s->update) stmt(s->update, cont, d + 2);
                if (s->k == Stmt::Loop) {
                    // continuing sees the body's declarations in WGSL; they are rare, so they are refused rather than hoisted
                    push();
                    for (const StmtP &c : s->cont) {
                        if (c->k == Stmt::BreakIf) {
                            Ty ct = check(c->e);
                            if (ct != scalar(S_BOOL)) invalid(c->e->line, c->e->col, "break if needs bool");
                            cont += ind(d + 2) + "if (" + code(c->e) + ") break;\n";
                        } else {
                            stmt(c, cont, d + 2);
                        }
                    }
                    pop();
                }
                pop();
                o += ind(d) + "{\n" + pre + ind(d + 1) + "for (;;) {\n";
                if (!cond.empty()) o += ind(d + 2) + "if (!(" + cond + ")) break;\n";
                o += ind(d + 2) + body + "\n" + ind(d + 2) + L + ":;\n" + cont + ind(d + 1) + "}\n" + ind(d) + "}\n";
                return;
            }
            case Stmt::Break:
                if (loops.empty()) invalid(s->line, s->col, "break outside a loop or switch");
                o += ind(d) + "break;\n";
                return;
            case Stmt::BreakIf:
                invalid(s->line, s->col, "break if outside continuing");
            case Stmt::Continue: {
                int lab = -1;
                for (auto it = loops.rbegin(); it != loops.rend(); ++it) if (*it >= 0) { lab = *it; break; }
                if (lab < 0) invalid(s->line, s->col, "continue outside a loop");
                o += ind(d) + "goto wg_cont_" + std::to_string(lab) + ";\n";
                return;
            }
            case Stmt::Return: {
                const Ty &r = cur_fn->ret;
                if (!s->e) {
                    if (r.k != Ty::Void) invalid(s->line, s->col, "return needs a value of type " + tname(r));
                    o += ind(d) + "return;\n";
                    return;
                }
                if (r.k == Ty::Void) invalid(s->line, s->col, "this function returns no value");
                check(s->e);
                conv(s->e, r);
                o += ind(d) + "return " + value(s->e) + ";\n";
                return;
            }
            case Stmt::Discard:
                if (cur_stage == "vertex") invalid(s->line, s->col, "discard in a vertex shader");
                o += ind(d) + "{ ctx.discarded = true; return" + (cur_fn->ret.k == Ty::Void ? std::string("") : " " + cty(cur_fn->ret) + "{}") + "; }\n";
                return;
            case Stmt::CallS: {
                check(s->e);
                o += ind(d) + code(s->e) + ";\n";
                return;
            }
        }
    }
};

// ------------------------------------------------------------------------------------------------------- the whole module
struct Varying {
    int location;
    Ty ty;
    int slot;
    int interp;    // 0 perspective, 1 linear, 2 flat
};

int interp_of(const Attrs &a, const Ty &t, int line, int col) {
    const Attr *i = find_attr(a, "interpolate");
    int k = 0;
    if (i && !i->args.empty()) {
        if (i->args[0] == "perspective") k = 0;
        else if (i->args[0] == "linear") k = 1;
        else if (i->args[0] == "flat") k = 2;
        else invalid(i->line, i->col, "unknown interpolation " + i->args[0]);
    }
    if ((t.s == S_I32 || t.s == S_U32) && k != 2) invalid(line, col, "an integer varying must be @interpolate(flat)");
    return k;
}

Translation run(const std::string &src) {
    Parser ps;
    ps.t = lex(src);
    ps.module();
    Module &m = ps.m;
    Checker ck(m);
    for (const StructDecl &s : m.structs) {
        if (ck.struct_ids.count(s.name)) invalid(s.line, s.col, "redeclaration of struct " + s.name);
        ck.struct_ids[s.name] = (int)ck.structs.size();
        StructInfo si;
        si.name = s.name; si.line = s.line; si.col = s.col;
        ck.structs.push_back(si);
    }
    for (const AliasDecl &a : m.aliases) {
        if (ck.struct_ids.count(a.name) || ck.aliases.count(a.name)) invalid(a.line, a.col, "redeclaration of '" + a.name + "'");
        ck.aliases[a.name] = &a;
    }
    ck.push();   // module scope
    // module constants, in order (a constant may use only those before it)
    for (const ConstDecl &c : m.consts) {
        Ty t = ck.check(c.init);
        Sym sym;
        sym.k = Sym::ModConst;
        if (c.ty) {
            Ty d = ck.resolve(c.ty);
            ck.conv(c.init, d);
            t = d;
        }
        sym.ty = t;
        if (c.init->has_cv && !c.ty) {
            sym.has_cv = true; sym.cv = c.init->cv;
        } else {
            sym.code = "u_" + c.name + "()";
            ck.const_int(sym, c.init);
            if (c.init->code.find("ctx") != std::string::npos) invalid(c.line, c.col, "a module constant must be a constant expression");
            ck.out_consts += "__device__ inline " + ck.cty(t) + " u_" + c.name + "() { return " + ck.value(c.init) + "; }\n";
        }
        if (ck.aliases.count(c.name)) invalid(c.line, c.col, "redeclaration of '" + c.name + "'");
        ck.const_value(sym, c.init);
        ck.declare(c.name, sym, c.line, c.col);
    }
    for (size_t i = 0; i < ck.structs.size(); i++) ck.resolve_struct((int)i);
    for (const AliasDecl &a : m.aliases) ck.resolve(a.ty);   // an unknown target or a cycle, even when unused
    // globals: the header's and the user's uniform
    const Global *g_tex = nullptr, *g_samp = nullptr, *g_base = nullptr;
    for (const Global &g : m.globals) {
        const Attr *ga = find_attr(g.attrs, "group"), *ba = find_attr(g.attrs, "binding");
        int group = ga && !ga->args.empty() ? atoi(ga->args[0].c_str()) : -1, binding = ba && !ba->args.empty() ? atoi(ba->args[0].c_str()) : -1;
        if (!g.ty && !(g.space == "private" && g.init)) invalid(g.line, g.col, "a module variable needs a type");
        if (group == 1 && binding == 0 && g.space != "uniform")
            invalid(g.line, g.col, "the user binding at group(1) binding(0) must be var<uniform> (UserBindingNotUniform)");
        if (g.space == "storage") unsupported(g.line, g.col, "storage buffers (var<storage>)");
        if (g.space == "workgroup") unsupported(g.line, g.col, "var<workgroup>");
        if (g.space == "push_constant")
            invalid(g.line, g.col, "var<push_constant> is not accepted: base_params is var<immediate>, as the shader header declares it");
        if (g.init && g.space != "private") unsupported(g.line, g.col, "initialised module variables");
        Ty t = g.ty ? ck.resolve(g.ty) : Ty();
        Sym sym;
        sym.ty = t;
        if (g.space == "private") {   // per-invocation state in wg_ctx, reset as each vs_main / fs_main invocation begins
            if (ga || ba) invalid(g.line, g.col, "var<private> takes no binding");
            std::string init;
            if (g.init) {
                Ty it = ck.check(g.init);
                if (g.ty) ck.conv(g.init, t);
                else { ck.conv_default(g.init); t = concrete(it); }
                init = ck.value(g.init);
                if (init.find("ctx") != std::string::npos) invalid(g.init->line, g.init->col, "a var<private> initializer must be a const-expression");
            }
            if (t.k == Ty::Tex || t.k == Ty::Samp || t.k == Ty::TexArr || t.k == Ty::Void) invalid(g.line, g.col, "a var<private> cannot hold " + ck.tname(t));
            sym.k = Sym::Private; sym.ty = t; sym.mut = true; sym.code = "ctx.pv.u_" + g.name;
            ck.has_private = true;
            ck.out_private += "    " + ck.cty(t) + " u_" + g.name + ";\n";
            if (g.init) ck.out_private_init += "    ctx.pv.u_" + g.name + " = " + init + ";\n";
        } else if (g.space == "immediate") {
            if (group >= 0 || binding >= 0) invalid(g.line, g.col, "var<immediate> takes no binding");
            if (g_base) invalid(g.line, g.col, "a second var<immediate>");
            g_base = &g;
            sym.k = Sym::Base; sym.code = "ctx.base";
        } else if (group == 1 && binding == 0) {
            if (g.space != "uniform") invalid(g.line, g.col, "the user binding at group(1) binding(0) must be var<uniform> (UserBindingNotUniform)");
            uint32_t al, sz;
            ck.layout(t, al, sz, g.line, g.col);
            ck.uniform = &g;
            ck.uniform_ty = t;
            sym.k = Sym::Uniform; sym.code = "0";
        } else if (group == 0 && binding == 0 && g.space.empty()) {
            g_tex = &g;
            sym.k = Sym::Textures;
        } else if (group == 2 && binding == 0 && g.space.empty()) {
            g_samp = &g;
            sym.k = Sym::Sampler; sym.code = "wg_sampler{}";
        } else if (g.space == "uniform") {
            unsupported(g.line, g.col, "uniform bindings other than group(1) binding(0)");
        } else if (g.space.empty() && group >= 0) {
            if (t.k == Ty::Tex || t.k == Ty::TexArr || t.k == Ty::Samp) unsupported(g.line, g.col, "texture and sampler bindings other than the header's");
            invalid(g.line, g.col, "a module variable needs an address space");
        } else {
            invalid(g.line, g.col, "unknown address space '" + g.space + "'");
        }
        if (ck.lookup(g.name) || ck.aliases.count(g.name)) invalid(g.line, g.col, "redeclaration of '" + g.name + "'");
        ck.declare(g.name, sym, g.line, g.col);
    }
    // validate_contains_header: the header's globals, at their spaces and bindings, with equivalent types (matched by
    // space and binding, not by name, as the reference does)
    auto global_missing = [&](const char *what) { invalid(1, 1, std::string("the shader header's global ") + what + " is missing (GlobalNotFound)"); };
    if (!g_tex) global_missing("textures: binding_array<texture_2d<f32>, 16> at @group(0) @binding(0)");
    if (!g_samp) global_missing("sampler_: sampler at @group(2) @binding(0)");
    if (!g_base) global_missing("base_params: BaseShaderParameters as var<immediate>");
    {
        Ty t = ck.lookup(g_tex->name)->ty;
        if (t.k != Ty::TexArr || t.n != 16) invalid(g_tex->line, g_tex->col, g_tex->name + " has type " + ck.tname(t) + ", expected binding_array<texture_2d<f32>, 16> (GlobalBadType)");
        t = ck.lookup(g_samp->name)->ty;
        if (t.k != Ty::Samp) invalid(g_samp->line, g_samp->col, g_samp->name + " has type " + ck.tname(t) + ", expected sampler (GlobalBadType)");
        t = ck.lookup(g_base->name)->ty;
        bool ok = t.k == Ty::Struct && ck.structs[t.sid].name == "BaseShaderParameters";
        if (ok) {
            const auto &f = ck.structs[t.sid].fields;
            const std::pair<const char *, Ty> want[4] = {{"plane_id", scalar(S_I32)}, {"time", scalar(S_F32)},
                                                         {"output_resolution", vec(S_U32, 2)}, {"texture_count", scalar(S_U32)}};
            ok = f.size() == 4;
            for (size_t i = 0; ok && i < 4; i++) ok = f[i].name == want[i].first && f[i].ty == want[i].second && f[i].attrs.empty();
        }
        if (!ok) invalid(g_base->line, g_base->col, g_base->name + " must be the header's struct BaseShaderParameters { plane_id: i32, time: f32, "
                                                    "output_resolution: vec2<u32>, texture_count: u32 } (GlobalBadType)");
    }
    // functions: signatures first (a function may call one declared after it)
    const FnDecl *vs = nullptr, *fs = nullptr;
    for (const FnDecl &f : m.fns) {
        if (ck.fns.count(f.name) || ck.struct_ids.count(f.name) || ck.aliases.count(f.name) || ck.lookup(f.name))
            invalid(f.line, f.col, "redeclaration of '" + f.name + "'");
        if (find_attr(f.attrs, "compute")) unsupported(f.line, f.col, "compute shaders");
        const bool entry = find_attr(f.attrs, "vertex") || find_attr(f.attrs, "fragment");
        FnInfo fi;
        fi.d = &f;
        for (const Param &p : f.params) {   // a helper may take a texture or the sampler; an entry point may not
            Ty t = ck.resolve(p.ty);
            if (t.k == Ty::TexArr) unsupported(f.line, f.col, "binding array parameters");
            if ((t.k == Ty::Tex || t.k == Ty::Samp) && entry) invalid(p.line, p.col, "an entry point cannot take " + ck.tname(t));
            fi.params.push_back(t);
        }
        fi.ret = f.ret ? ck.resolve(f.ret) : Ty();
        if (fi.ret.k == Ty::Tex || fi.ret.k == Ty::Samp || fi.ret.k == Ty::TexArr) invalid(f.ret->line, f.ret->col, "a function cannot return " + ck.tname(fi.ret));
        fi.cname = "fn_" + f.name;
        if (find_attr(f.attrs, "vertex")) {
            if (f.name == "vs_main") vs = &f;
        }
        if (find_attr(f.attrs, "fragment")) {
            if (f.name == "fs_main") fs = &f;
        }
        ck.fns[f.name] = fi;
    }
    // validate_vertex_input: vs_main takes exactly one VertexInput equivalent to the header's
    if (!vs) invalid(1, 1, "no @vertex fn vs_main (VertexShaderNotFound)");
    if (vs->params.size() != 1) invalid(vs->line, vs->col, "vs_main takes " + std::to_string(vs->params.size()) + " arguments, expected 1 (VertexShaderBadArgumentAmount)");
    {
        const Ty &vi = ck.fns["vs_main"].params[0];
        bool ok = vi.k == Ty::Struct && ck.structs[vi.sid].name == "VertexInput";
        if (!ok) invalid(vs->line, vs->col, "vs_main's argument must be the header's VertexInput (VertexShaderBadInputTypeName)");
        const auto &f = ck.structs[vi.sid].fields;
        ok = f.size() == 2 && f[0].name == "position" && f[0].ty == vec(S_F32, 3) && f[1].name == "tex_coords" && f[1].ty == vec(S_F32, 2);
        for (size_t i = 0; ok && i < 2; i++) {
            const Attr *l = find_attr(f[i].attrs, "location");
            ok = l && l->args.size() == 1 && l->args[0] == std::to_string(i) && f[i].attrs.size() == 1;
        }
        if (!ok) invalid(vs->line, vs->col, "VertexInput must be { @location(0) position: vec3<f32>, @location(1) tex_coords: vec2<f32> } (VertexShaderBadInput)");
    }
    if (!fs) invalid(1, 1, "no @fragment fn fs_main");
    for (const StmtP &a : m.asserts) ck.const_assert(a);
    // function bodies
    for (const FnDecl &f : m.fns) {
        FnInfo &fi = ck.fns[f.name];
        ck.cur_fn = &fi;
        ck.cur_stage = find_attr(f.attrs, "vertex") ? "vertex" : find_attr(f.attrs, "fragment") ? "fragment" : "";
        std::string sig = "__device__ " + (fi.ret.k == Ty::Void ? std::string("void") : ck.cty(fi.ret)) + " " + fi.cname + "(wg_ctx &ctx";
        for (size_t i = 0; i < f.params.size(); i++) sig += ", " + ck.cty(fi.params[i]) + " u_" + f.params[i].name;
        sig += ")";
        ck.out_protos += sig + ";\n";
        ck.push();
        for (size_t i = 0; i < f.params.size(); i++) {
            Sym s;
            s.k = Sym::Param; s.ty = fi.params[i]; s.code = "u_" + f.params[i].name;
            ck.declare(f.params[i].name, s, f.line, f.col);
        }
        std::string body = sig + " {\n";
        ck.stmts(f.body, body, 1);
        if (fi.ret.k != Ty::Void) body += "    return " + ck.cty(fi.ret) + "{};\n";   // unreachable in a valid module
        body += "}\n";
        ck.pop();
        ck.out_bodies += body;
    }
    // textureSampleBias is a fragment-stage builtin: refused in vs_main and in every function vs_main reaches
    {
        std::set<std::string> seen;
        std::function<void(const std::string &)> vertex_ok = [&](const std::string &fn) {
            if (!seen.insert(fn).second) return;
            const FnInfo &fi = ck.fns[fn];
            if (fi.frag_line) invalid(fi.frag_line, fi.frag_col, "textureSampleBias is only allowed in the fragment stage, and vs_main reaches it");
            for (const std::string &c : fi.calls) vertex_ok(c);
        };
        vertex_ok("vs_main");
    }
    // the stage interface: vs_main's output and fs_main's input
    const FnInfo &vsi = ck.fns["vs_main"], &fsi = ck.fns["fs_main"];
    std::vector<Varying> vary;
    std::string vs_store;
    int nvary = 0;
    auto vary_store = [&](const Ty &t, const std::string &v, int slot) {
        std::string s;
        int n = t.k == Ty::Vec ? t.n : 1;
        for (int k = 0; k < n; k++) {
            std::string c = t.k == Ty::Vec ? v + ".v[" + std::to_string(k) + "]" : v;
            s += "    vary[" + std::to_string(slot + k) + "] = " + (t.s == S_F32 ? c : "__uint_as_float((unsigned)" + c + ")") + ";\n";
        }
        return s;
    };
    auto varying_ok = [&](const Ty &t, int line, int col) {
        if (!((t.k == Ty::Scalar || t.k == Ty::Vec) && t.s != S_BOOL)) invalid(line, col, "a varying must be a numeric scalar or vector");
    };
    bool has_pos = false;
    if (vsi.ret.k == Ty::Struct) {
        for (const FieldInfo &f : ck.structs[vsi.ret.sid].fields) {
            const Attr *b = find_attr(f.attrs, "builtin"), *l = find_attr(f.attrs, "location");
            if (b && b->args.size() == 1 && b->args[0] == "position") {
                if (f.ty != vec(S_F32, 4)) invalid(vs->line, vs->col, "@builtin(position) must be vec4<f32>");
                has_pos = true;
                vs_store += "    for (int k = 0; k < 4; k++) pos[k] = o.m_" + f.name + ".v[k];\n";
            } else if (l && l->args.size() == 1) {
                varying_ok(f.ty, vs->line, vs->col);
                Varying v;
                v.location = atoi(l->args[0].c_str());
                v.ty = f.ty;
                v.slot = nvary;
                v.interp = interp_of(f.attrs, f.ty, vs->line, vs->col);
                for (const Varying &w : vary) if (w.location == v.location) invalid(vs->line, vs->col, "duplicate @location in vs_main's output");
                vary.push_back(v);
                vs_store += vary_store(f.ty, "o.m_" + f.name, nvary);
                nvary += f.ty.k == Ty::Vec ? f.ty.n : 1;
            } else {
                invalid(vs->line, vs->col, "every member of vs_main's output needs @location or @builtin(position)");
            }
        }
    } else if (vsi.ret == vec(S_F32, 4)) {
        const Attr *b = find_attr(vs->ret_attrs, "builtin");
        if (!b || b->args.size() != 1 || b->args[0] != "position") invalid(vs->line, vs->col, "vs_main's vec4 result needs @builtin(position)");
        has_pos = true;
        vs_store += "    for (int k = 0; k < 4; k++) pos[k] = o.v[k];\n";
    }
    if (!has_pos) invalid(vs->line, vs->col, "vs_main must output @builtin(position)");
    if (nvary > 64) unsupported(vs->line, vs->col, "more than 64 varying components");
    // fs_main's input: each argument a struct of bound members or a bound value
    std::string fs_args, fs_pre;
    int interp[64] = {0};
    std::vector<bool> used(64, false);
    auto bind_in = [&](const Ty &t, const Attrs &a, const std::string &dst) -> std::string {
        const Attr *b = find_attr(a, "builtin"), *l = find_attr(a, "location");
        if (b && b->args.size() == 1 && b->args[0] == "position") {
            if (t != vec(S_F32, 4)) invalid(fs->line, fs->col, "@builtin(position) must be vec4<f32>");
            return "    " + dst + " = wv<float, 4>{{pos[0], pos[1], pos[2], pos[3]}};\n";
        }
        if (b && b->args.size() == 1 && b->args[0] == "front_facing") {
            if (t != scalar(S_BOOL)) invalid(fs->line, fs->col, "@builtin(front_facing) must be bool");
            return "    " + dst + " = true;\n";   // back faces are culled
        }
        if (b) unsupported(fs->line, fs->col, "@builtin(" + (b->args.empty() ? std::string("") : b->args[0]) + ") in fs_main");
        if (!l || l->args.size() != 1) invalid(fs->line, fs->col, "every input of fs_main needs @location or @builtin");
        int loc = atoi(l->args[0].c_str());
        const Varying *v = nullptr;
        for (const Varying &w : vary) if (w.location == loc) v = &w;
        if (!v) invalid(fs->line, fs->col, "fs_main reads @location(" + l->args[0] + "), which vs_main does not write");
        if (v->ty != t) invalid(fs->line, fs->col, "@location(" + l->args[0] + ") has type " + ck.tname(v->ty) + " in vs_main and " + ck.tname(t) + " in fs_main");
        int k = interp_of(a, t, fs->line, fs->col);
        int n = t.k == Ty::Vec ? t.n : 1;
        std::string s;
        for (int j = 0; j < n; j++) {
            interp[v->slot + j] = k;
            std::string c = "vary[" + std::to_string(v->slot + j) + "]";
            if (t.s != S_F32) c = "(" + ck.cscalar(t.s) + ")__float_as_uint(" + c + ")";
            s += "    " + dst + (t.k == Ty::Vec ? ".v[" + std::to_string(j) + "]" : "") + " = " + c + ";\n";
        }
        return s;
    };
    for (size_t i = 0; i < fs->params.size(); i++) {
        const Ty &t = fsi.params[i];
        std::string nm = "in" + std::to_string(i);
        fs_pre += "    " + ck.cty(t) + " " + nm + "{};\n";
        if (t.k == Ty::Struct) {
            for (const FieldInfo &f : ck.structs[t.sid].fields) fs_pre += bind_in(f.ty, f.attrs, nm + ".m_" + f.name);
        } else {
            fs_pre += bind_in(t, fs->params[i].attrs, nm);
        }
        fs_args += ", " + nm;
    }
    // fs_main's result: @location(0) vec4<f32>, or a struct whose only member is one
    std::string fs_result;
    {
        auto location0 = [](const Attrs &a) {
            const Attr *l = find_attr(a, "location");
            return l && l->args.size() == 1 && l->args[0] == "0";
        };
        bool ok = fsi.ret == vec(S_F32, 4) && location0(fs->ret_attrs);
        if (fsi.ret.k == Ty::Struct && fs->ret_attrs.empty()) {
            const auto &f = ck.structs[fsi.ret.sid].fields;
            ok = f.size() == 1 && f[0].ty == vec(S_F32, 4) && f[0].attrs.size() == 1 && location0(f[0].attrs);
            if (ok) fs_result = ".m_" + f[0].name;
        }
        if (!ok) unsupported(fs->line, fs->col, "fs_main results other than @location(0) vec4<f32>");
    }
    // the translation
    Translation tr;
    std::string out = "// translated from WGSL\n" + ck.out_structs;
    const Ty base = ck.lookup(g_base->name)->ty;
    if (!ck.out_private.empty()) out += "struct wg_private {\n" + ck.out_private + "};\n";
    out += "struct wg_ctx {\n    " + ck.cty(base) + " base;\n    const unsigned char *params;\n    wg_textures tex;\n    bool discarded;\n" +
           (ck.out_private.empty() ? "" : "    wg_private pv;\n") + "};\n";
    if (ck.uniform) {
        ck.load(ck.uniform_ty, "p");   // the loaders of the uniform's composite types
        uint32_t al, sz;
        ck.layout(ck.uniform_ty, al, sz, 0, 0);
        tr.uniform_size = sz;
    }
    out += ck.out_loaders + ck.out_consts + ck.out_protos;
    // the var<private> state starts at its initial value (or zero) in every invocation
    std::string reset;
    if (!ck.out_private.empty()) {
        out += "__device__ inline void wg_private_reset(wg_ctx &ctx) {\n    ctx.pv = wg_private{};\n" + ck.out_private_init + "}\n";
        reset = "    wg_private_reset(ctx);\n";
    }
    out += ck.out_bodies;
    const Ty &vin = vsi.params[0];
    out += "#define WG_NVARY " + std::to_string(nvary) + "\n";
    out += "__device__ const unsigned char wg_interp[" + std::to_string(std::max(1, nvary)) + "] = {";
    for (int i = 0; i < std::max(1, nvary); i++) out += (i ? ", " : "") + std::to_string(interp[i]);
    out += "};\n";
    out += "__device__ inline void wg_base(wg_ctx &ctx, int plane, float time, unsigned w, unsigned h, unsigned n) {\n"
           "    ctx.base.m_plane_id = plane;\n    ctx.base.m_time = time;\n"
           "    ctx.base.m_output_resolution = wv<unsigned, 2>{{w, h}};\n    ctx.base.m_texture_count = n;\n}\n";
    out += "// the plane mesh (plane.rs): position, tex_coords\n"
           "__device__ inline void wg_vertex(wg_ctx &ctx, int vid, float *pos, float *vary) {\n"
           "    const float P[4][5] = {{1.0f, -1.0f, 0.0f, 1.0f, 1.0f}, {1.0f, 1.0f, 0.0f, 1.0f, 0.0f},\n"
           "                           {-1.0f, 1.0f, 0.0f, 0.0f, 0.0f}, {-1.0f, -1.0f, 0.0f, 0.0f, 1.0f}};\n"
           "    " + ck.cty(vin) + " in;\n"
           "    in.m_position = wv<float, 3>{{P[vid][0], P[vid][1], P[vid][2]}};\n"
           "    in.m_tex_coords = wv<float, 2>{{P[vid][3], P[vid][4]}};\n" + reset +
           "    const " + ck.cty(vsi.ret) + " o = fn_vs_main(ctx, in);\n" + vs_store +
           "    (void)vary;\n}\n";
    out += "__device__ inline bool wg_fragment(wg_ctx &ctx, const float *pos, const float *vary, float4 &out) {\n" + fs_pre + reset +
           "    (void)vary;\n    ctx.discarded = false;\n    const wv<float, 4> r = fn_fs_main(ctx" + fs_args + ")" + fs_result + ";\n"
           "    out = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);\n    return !ctx.discarded;\n}\n";
    tr.cuda = out;
    // the parameter type: validate_params' view of the uniform's WGSL type
    if (ck.uniform) {
        std::function<ShaderParamType(const Ty &, const std::string &)> pt = [&](const Ty &t, const std::string &name) {
            ShaderParamType p;
            p.name = name;
            switch (t.k) {
                case Ty::Scalar: p.kind = t.s == S_F32 ? SMR_SHADER_PARAM_F32 : t.s == S_U32 ? SMR_SHADER_PARAM_U32 : SMR_SHADER_PARAM_I32; break;
                case Ty::Vec:
                    p.kind = kShaderParamVector;
                    p.length = (uint32_t)t.n;
                    p.items.push_back(pt(scalar(t.s), ""));
                    break;
                case Ty::Mat:
                    p.kind = kShaderParamMatrix;
                    p.length = (uint32_t)t.m;   // rows
                    p.items.push_back(pt(vec(S_F32, t.n), ""));
                    break;
                case Ty::Arr:
                    p.kind = SMR_SHADER_PARAM_LIST;
                    p.length = (uint32_t)t.n;
                    p.items.push_back(pt(*t.el, ""));
                    break;
                default:
                    p.kind = SMR_SHADER_PARAM_STRUCT;
                    for (const FieldInfo &f : ck.structs[t.sid].fields) p.items.push_back(pt(f.ty, f.name));
                    break;
            }
            return p;
        };
        tr.param_type = pt(ck.uniform_ty, "");
    }
    return tr;
}

}  // namespace

Translation translate(const std::string &source) {
    try {
        return run(source);
    } catch (const Fail &f) {
        Translation t;
        t.status = f.status;
        t.error = "WGSL " + f.msg;
        return t;
    }
}

}  // namespace wgsl
}  // namespace smr
