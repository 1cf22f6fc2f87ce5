// Lua -> C++/CUDA transpiler for lens scripts.  See lua_transpile.h.
#include "lua_transpile.h"

#include <cmath>
#include <cstdio>
#include <map>
#include <set>
#include <sstream>

#include "minilua/minilua_ast.h"

using namespace minilua;

namespace blinky {

namespace {

struct Fail {
    std::string why;
};
[[noreturn]] void fail(const std::string &why, int line = 0) {
    std::ostringstream o;
    if (line) o << "line " << line << ": ";
    o << why;
    throw Fail{o.str()};
}

enum class VT { Num, Bool, Arr };

struct EOut {
    std::string code;
    VT type = VT::Num;
    bool tainted = false;
    int arr_size = 0;        // VT::Arr: number of elements
    std::string arr_name;    // VT::Arr
};

struct BuiltinInfo {
    std::string name;
    bool libm;  // result may differ between glibc and CUDA in the last bits
};

std::string num_literal(double d) {
    if (d != d) return "LT_NAN";
    if (std::isinf(d)) return d > 0 ? "LT_INF" : "(-LT_INF)";
    char b[64];
    snprintf(b, sizeof b, "%a", d);  // exact hexadecimal floating literal (C++17)
    return std::string("(") + b + ")";
}

struct LocalInfo {
    std::string cname;
    VT type = VT::Num;
    int arr_size = 0;
    bool tainted = false;
};

struct FuncInfo {
    const Function *fn = nullptr;
    std::string cname;
    int arity = -1;
    std::vector<int> res_types;  // per result: -1 unknown yet, else static_cast<int>(VT::Num / VT::Bool)
    std::vector<bool> exact_params;  // per parameter: a plain double (only entry points have such parameters)
    bool in_progress = false;
    bool done = false;
    std::string code;
};

class Transpiler {
public:
    explicit Transpiler(State &L) : L_(L) { collect_builtins(); }

    // entry: the lens function (nullptr: globe_plate alone); globe_plate (may be nullptr) joins the same
    // translation unit: one function table, one set of constant tables, one set of script-level slots
    TranspileResult run(const Value *entry, int nparams, int nresults, const char *what, const Value *globe_plate) {
        TranspileResult r;
        bool in_globe_plate = false;
        try {
            const std::string name = what;
            const Function *fn = entry ? check_entry(*entry, nparams, name) : nullptr;
            const Function *gp = nullptr;
            if (globe_plate) {
                in_globe_plate = true;
                gp = check_entry(*globe_plate, 3, "globe_plate");
                in_globe_plate = false;
            }
            // pass 1: which script-level variables do the functions assign?
            std::set<const Function *> seen;
            if (fn) {
                scan_function(fn, seen);
                entry_fns_.insert(fn);
            }
            if (gp) {
                in_globe_plate = true;
                scope_ = "globe_plate";
                scan_function(gp, seen);
                entry_fns_.insert(gp);
                scope_ = "lens";
                in_globe_plate = false;
            }
            FuncInfo *fip = nullptr;
            if (fn) {
                FuncInfo &fi = gen_function(fn);
                if (fi.arity != nresults) fail(name + " must return " + (nresults == 3 ? std::string("three") : std::to_string(nresults)) + " numbers (or nil)");
                for (int t : fi.res_types)
                    if (t == static_cast<int>(VT::Bool)) fail(name + " must return numbers, not booleans");
                fip = &fi;
            }
            FuncInfo *gip = nullptr;
            if (gp) {
                in_globe_plate = true;
                scope_ = "globe_plate";
                FuncInfo &gi = gen_function(gp);
                for (int t : gi.res_types)
                    if (t == static_cast<int>(VT::Bool)) fail("globe_plate must return numbers, not booleans");
                scope_ = "lens";
                in_globe_plate = false;
                gip = &gi;
            }
            std::ostringstream o;
            o << "LT_FN void lt_init_mut(Ctx &c) {\n    (void)c;\n";
            for (size_t i = 0; i < mutable_init_.size(); ++i) o << "    c.mg[" << i << "] = LtD(" << num_literal(mutable_init_[i]) << ");\n";
            o << "}\n";
            if (mutable_init_.size() > 32) fail(std::string("too many script-level variables are assigned by the ") + (gp ? "lens and globe_plate" : "lens"));
            o << tables_.str();
            for (const std::string &c : order_) o << c << "\n";
            if (fip) {
                o << "LT_FN bool lt_entry(Ctx &c";
                for (int i = 0; i < nparams; ++i) o << ", double a" << i;
                o << ", LtD *r) { return " << fip->cname << "(c";
                for (int i = 0; i < nparams; ++i) o << ", a" << i;
                o << ", r); }\n";
            }
            if (gip) emit_globe_plate_entry(o, *gip);
            r.ok = true;
            r.source = o.str();
            r.num_functions = static_cast<int>(order_.size());
            r.num_mutable = static_cast<int>(mutables_.size());
        } catch (Fail &f) {
            r.ok = false;
            r.error = in_globe_plate ? "globe_plate: " + f.why : f.why;
        }
        return r;
    }

private:
    const Function *check_entry(const Value &entry, int nparams, const std::string &name) {
        if (!entry.is_function()) fail(name + " is not a function");
        const Function *fn = static_cast<const Function *>(entry.obj());
        if (fn->cfn) fail(name + " is a C function");
        if (fn->proto->nparams != nparams || fn->proto->is_vararg) fail(name + " must take exactly " + std::to_string(nparams) + " arguments");
        return fn;
    }

    // ray_to_plate_index with a globe_plate script (fisheye.c:2027-2033, :1634-1651): the LAST value returned
    // counts; none, nil or a non-number is plate -1; a number d becomes (int)(ptrdiff_t)d (lua_tointeger).
    // That conversion is a decision: it is flagged when an integer lies within d's error bound, and when d is
    // NaN, infinite or outside int range, where x86 and CUDA convert differently.
    void emit_globe_plate_entry(std::ostringstream &o, const FuncInfo &gi) {
        const int k = gi.arity;
        o << "#define LT_HAS_GLOBE_PLATE 1\n";
        o << "LT_FN int lt_plate_int(Ctx &c, LtD x) {\n"
             "    if (!(fabs(x.v) < 2147483000.0)) { c.flag |= LT_RISK_NEAR; return -1; }\n"
             "    if (!(x.e == 0.0)) {\n"
             "        const double n = rint(x.v);\n"
             "        if (!(fabs(x.v - n) > 2.0 * x.e)) c.flag |= LT_RISK_NEAR;\n"
             "    }\n"
             "    return (int)x.v;\n"
             "}\n";
        o << "LT_FN bool lt_globe_plate(Ctx &c, double x, double y, double z, int *plate) {\n";
        o << "    LtD r[" << std::max(1, k) << "];\n";
        o << "    *plate = -1;\n";
        if (k == 0) {
            o << "    " << gi.cname << "(c, x, y, z, r);\n    return false;\n}\n";  // never returns a value
            return;
        }
        o << "    if (!" << gi.cname << "(c, x, y, z, r)) return false;\n";
        o << "    *plate = lt_plate_int(c, r[" << k - 1 << "]);\n";
        o << "    return true;\n}\n";
    }

    // ------------------------------------------------------------------ builtins
    void add_builtin(const Value &v, const std::string &name, bool libm) {
        if (v.is_function()) builtins_[v.obj()] = BuiltinInfo{name, libm};
    }
    void collect_builtins() {
        Value m = L_.get_global("math");
        if (m.is_table()) {
            Table *t = static_cast<Table *>(m.obj());
            static const struct { const char *n; bool libm; } kMath[] = {
                {"abs", false}, {"acos", true}, {"asin", true}, {"atan", true}, {"atan2", true}, {"ceil", false},
                {"cos", true}, {"cosh", true}, {"exp", true}, {"floor", false}, {"fmod", false}, {"log", true},
                {"log10", true}, {"max", false}, {"min", false}, {"modf", false}, {"pow", true}, {"sin", true},
                {"sinh", true}, {"sqrt", false}, {"tan", true}, {"tanh", true}, {"deg", false}, {"rad", false}};
            for (auto &e : kMath) add_builtin(t->get_str(e.n), std::string("math.") + e.n, e.libm);
        }
        add_builtin(L_.get_global("latlon_to_ray"), "latlon_to_ray", true);
        add_builtin(L_.get_global("ray_to_latlon"), "ray_to_latlon", true);
        add_builtin(L_.get_global("plate_to_ray"), "plate_to_ray", false);
        add_builtin(L_.get_global("print"), "print", false);
    }

    // ------------------------------------------------------------------ value resolution
    // the CURRENT value a Global/Upval expression denotes inside closure `fn`
    Value current_value(const Function *fn, const Expr *e, const void **identity) {
        if (e->k == EK::Global) {
            *identity = reinterpret_cast<const void *>(static_cast<uintptr_t>(e->id) + 1);  // ids are small ints
            return L_.global_slot(e->id);
        }
        Box *b = fn->upvals[static_cast<size_t>(e->id)];
        *identity = b;
        return b->v;
    }

    // static resolution of a callee / table expression to a runtime Value (no side effects)
    bool static_value(const Function *fn, const Expr *e, Value *out) {
        const void *id;
        switch (e->k) {
            case EK::Global:
            case EK::Upval: *out = current_value(fn, e, &id); return true;
            case EK::Paren: return static_value(fn, e->l, out);
            case EK::Index: {
                Value t;
                if (!static_value(fn, e->l, &t) || !t.is_table()) return false;
                if (e->r->k == EK::String) {
                    *out = static_cast<Table *>(t.obj())->get(L_.kstr(e->r->id));
                    return true;
                }
                return false;
            }
            default: return false;
        }
    }

    // ------------------------------------------------------------------ pass 1: assigned script-level variables
    void scan_function(const Function *fn, std::set<const Function *> &seen) {
        if (!seen.insert(fn).second) return;
        scan_block(fn, fn->proto->body, seen);
    }
    void scan_block(const Function *fn, const Block *b, std::set<const Function *> &seen) {
        for (const Stmt *s : b->stmts) scan_stmt(fn, s, seen);
    }
    void note_mutable(const Function *fn, const Expr *target) {
        const void *id;
        Value cur = current_value(fn, target, &id);
        if (mutables_.count(id)) return;
        if (cur.is_nil()) {
            // a cache variable that starts out unset: NaN compares unequal to everything, like nil
            mutables_[id] = static_cast<int>(mutable_init_.size());
            mutable_init_.push_back(std::nan(""));
            return;
        }
        if (!cur.is_number()) {
            fail("the " + scope_ + " assigns script-level variable '" + var_name(fn, target) + "' whose current value is not a number", target->line);
        }
        mutables_[id] = static_cast<int>(mutable_init_.size());
        mutable_init_.push_back(cur.num());
    }
    std::string var_name(const Function *fn, const Expr *e) {
        if (e->k == EK::Global) return L_.universe()->global_names[static_cast<size_t>(e->id)];
        if (e->k == EK::Upval) return fn->proto->upvals[static_cast<size_t>(e->id)].name;
        return "?";
    }
    void scan_expr(const Function *fn, const Expr *e, std::set<const Function *> &seen) {
        if (!e) return;
        if (e->k == EK::Function) fail("closures created inside the " + scope_ + " are not supported", e->line);
        if (e->k == EK::Call) {
            Value callee;
            if (static_value(fn, e->l, &callee) && callee.is_function()) {
                const Function *cf = static_cast<const Function *>(callee.obj());
                if (!cf->cfn) scan_function(cf, seen);
            }
        }
        scan_expr(fn, e->l, seen);
        scan_expr(fn, e->r, seen);
        for (const Expr *x : e->list) scan_expr(fn, x, seen);
        for (const Expr *x : e->keys) scan_expr(fn, x, seen);
        for (const Expr *x : e->vals) scan_expr(fn, x, seen);
    }
    void scan_stmt(const Function *fn, const Stmt *s, std::set<const Function *> &seen) {
        for (const Expr *t : s->targets) {
            if (t->k == EK::Global || t->k == EK::Upval) note_mutable(fn, t);
            else if (t->k == EK::Index) scan_expr(fn, t, seen);
        }
        for (const Expr *e : s->exprs) scan_expr(fn, e, seen);
        scan_expr(fn, s->e, seen);
        for (const Expr *e : s->conds) scan_expr(fn, e, seen);
        if (s->body) scan_block(fn, s->body, seen);
        for (const Block *b : s->blocks) scan_block(fn, b, seen);
        if (s->k == SK::GenFor) fail("generic 'for ... in' is not supported", s->line);
        if (s->k == SK::LocalFunction) fail("local functions inside the " + scope_ + " are not supported", s->line);
        if (s->k == SK::Goto || s->k == SK::Label) fail("goto is not supported", s->line);
    }

    // ------------------------------------------------------------------ per-function generation state
    struct Gen {
        const Function *fn;
        FuncInfo *fi;
        std::map<const VarInfo *, LocalInfo> locals;
        std::ostringstream out;
        int indent = 1;
        int tmp = 0;
        bool is_entry = false;
    };

    void line(Gen &g, const std::string &s) {
        for (int i = 0; i < g.indent; ++i) g.out << "    ";
        g.out << s << "\n";
    }
    std::string new_tmp(Gen &g, const char *prefix = "t") { return std::string(prefix) + std::to_string(g.tmp++); }

    // ------------------------------------------------------------------ taint pre-pass (fixpoint)
    bool taint_expr(Gen &g, const Expr *e) {
        if (!e) return false;
        switch (e->k) {
            case EK::Nil: case EK::True: case EK::False: case EK::Number: case EK::String: return false;
            case EK::Local: {
                auto it = g.locals.find(e->var);
                return it != g.locals.end() && it->second.tainted;
            }
            case EK::Global:
            case EK::Upval: {
                const void *id;
                current_value(g.fn, e, &id);
                return mutables_.count(id) > 0;  // assigned by the lens: conservatively tainted
            }
            case EK::Call: {
                Value callee;
                if (static_value(g.fn, e->l, &callee) && callee.is_function()) {
                    auto b = builtins_.find(callee.obj());
                    if (b != builtins_.end()) {
                        const std::string &n = b->second.name;
                        if (b->second.libm) return n != "latlon_to_ray";  // its results pass through float32: exact again
                        if (n == "plate_to_ray" || n == "math.floor" || n == "math.ceil" || n == "print") return false;
                        bool t = false;
                        for (const Expr *a : e->list) t = taint_expr(g, a) || t;
                        return t;
                    }
                }
                return true;  // user function: results carry an error bound
            }
            case EK::Pow: return true;
            case EK::Eq: case EK::Ne: case EK::Lt: case EK::Le: case EK::Gt: case EK::Ge:
            case EK::And: case EK::Or: case EK::Not: case EK::Len: return false;
            case EK::Index: return taint_expr(g, e->l);
            default: {
                bool t = taint_expr(g, e->l);
                t = taint_expr(g, e->r) || t;
                for (const Expr *x : e->list) t = taint_expr(g, x) || t;
                return t;
            }
        }
    }
    bool taint_block(Gen &g, const Block *b) {
        bool changed = false;
        for (const Stmt *s : b->stmts) {
            auto mark = [&](const VarInfo *v, bool t) {
                LocalInfo &li = g.locals[v];
                if (t && !li.tainted) {
                    li.tainted = true;
                    changed = true;
                }
            };
            if (s->k == SK::Local) {
                bool any = false;
                for (const Expr *e : s->exprs) any = taint_expr(g, e) || any;
                for (size_t i = 0; i < s->vars.size(); ++i) {
                    bool t = i < s->exprs.size() && s->exprs.size() == s->vars.size() ? taint_expr(g, s->exprs[i]) : any;
                    mark(s->vars[i], t);
                }
            } else if (s->k == SK::Assign) {
                bool any = false;
                for (const Expr *e : s->exprs) any = taint_expr(g, e) || any;
                for (size_t i = 0; i < s->targets.size(); ++i) {
                    const Expr *t = s->targets[i];
                    bool tt = s->exprs.size() == s->targets.size() ? taint_expr(g, s->exprs[i]) : any;
                    if (t->k == EK::Local) mark(t->var, tt);
                    else if (t->k == EK::Index && t->l->k == EK::Local) mark(t->l->var, tt);
                }
            } else if (s->k == SK::NumFor) {
                mark(s->vars[0], false);  // the control variable is exact (see SK::NumFor)
            }
            if (s->body) changed = taint_block(g, s->body) || changed;
            for (const Block *bb : s->blocks) changed = taint_block(g, bb) || changed;
        }
        return changed;
    }

    // ------------------------------------------------------------------ function generation
    FuncInfo &gen_function(const Function *fn) {
        FuncInfo &fi = funcs_[fn];
        if (fi.done) return fi;
        if (fi.in_progress) fail("recursive functions are not supported (" + fn->proto->name + ")");
        fi.fn = fn;
        fi.in_progress = true;
        fi.cname = "lf" + std::to_string(funcs_.size()) + "_" + sanitize(fn->proto->name);
        if (fn->proto->is_vararg) fail("vararg functions are not supported (" + fn->proto->name + ")");
        fi.arity = compute_arity(fn, fn->proto->body);
        if (fi.arity < 0) fi.arity = 0;
        if (fi.arity > 8) fail("functions returning more than 8 values are not supported");

        Gen g;
        g.fn = fn;
        g.fi = &fi;
        g.is_entry = entry_fns_.count(fn) > 0;
        for (size_t i = 0; i < fn->proto->params.size(); ++i) {
            LocalInfo li;
            li.cname = "p" + std::to_string(i) + "_" + sanitize(fn->proto->params[i]->name);
            li.tainted = !g.is_entry;  // only the entry's (x, y) are known to be exact
            g.locals[fn->proto->params[i]] = li;
        }
        while (taint_block(g, fn->proto->body)) {
        }
        // the signature comes after the fixpoint: a parameter that is assigned an error-carrying value
        // inside the body has to be an LtD from the start
        std::ostringstream sig;
        sig << "LT_UFN bool " << fi.cname << "(Ctx &c";
        for (size_t i = 0; i < fn->proto->params.size(); ++i) {
            const LocalInfo &li = g.locals[fn->proto->params[i]];
            sig << (li.tainted ? ", LtD " : ", double ") << li.cname;
            fi.exact_params.push_back(!li.tainted);
        }
        sig << ", LtD *r) {";
        line(g, "(void)c; (void)r;");
        gen_block(g, fn->proto->body);
        line(g, "return false;");  // falling off the end returns nothing: nil
        fi.code = sig.str() + "\n" + g.out.str() + "}\n";
        fi.in_progress = false;
        fi.done = true;
        order_.push_back(fi.code);
        return fi;
    }

    static std::string sanitize(const std::string &s) {
        std::string o;
        for (char ch : s) o.push_back((isalnum(static_cast<unsigned char>(ch)) || ch == '_') ? ch : '_');
        return o.substr(0, 24);
    }

    // number of values a function returns (max over its return statements; `return nil` counts as the nil form)
    int compute_arity(const Function *fn, const Block *b) {
        int best = -1;
        for (const Stmt *s : b->stmts) {
            if (s->k == SK::Return) {
                int n = 0;
                if (s->exprs.size() == 1 && s->exprs[0]->k == EK::Nil) n = -1;  // nil form, does not fix the arity
                else {
                    for (size_t i = 0; i < s->exprs.size(); ++i) {
                        const Expr *e = s->exprs[i];
                        if (i + 1 == s->exprs.size() && e->k == EK::Call) n += call_arity(fn, e);
                        else n += 1;
                    }
                }
                if (n > best) best = n;
            }
            if (s->body) best = std::max(best, compute_arity(fn, s->body));
            for (const Block *bb : s->blocks) best = std::max(best, compute_arity(fn, bb));
        }
        return best;
    }

    int builtin_results(const std::string &name) {
        if (name == "latlon_to_ray" || name == "plate_to_ray") return 3;
        if (name == "ray_to_latlon" || name == "math.modf") return 2;
        if (name == "print") return 0;
        return 1;
    }

    int call_arity(const Function *fn, const Expr *call) {
        Value callee;
        if (!static_value(fn, call->l, &callee) || !callee.is_function()) fail("cannot resolve the function being called", call->line);
        auto b = builtins_.find(callee.obj());
        if (b != builtins_.end()) return builtin_results(b->second.name);
        const Function *cf = static_cast<const Function *>(callee.obj());
        if (cf->cfn) fail("call to an unsupported C function", call->line);
        return gen_function(cf).arity;
    }

    // ------------------------------------------------------------------ expressions
    EOut gen_expr(Gen &g, const Expr *e) {
        EOut o;
        switch (e->k) {
            case EK::Number: o.code = num_literal(e->num); return o;
            case EK::True: o.code = "true"; o.type = VT::Bool; return o;
            case EK::False: o.code = "false"; o.type = VT::Bool; return o;
            case EK::Nil: fail("nil values are not supported here", e->line);
            case EK::String: fail("strings are not supported", e->line);
            case EK::Vararg: fail("'...' is not supported", e->line);
            case EK::Function: fail("closures are not supported", e->line);
            case EK::Method: fail("method calls are not supported", e->line);
            case EK::Table: fail("table constructors are only supported in 'local t = {...}'", e->line);
            case EK::Concat: fail("string concatenation is not supported", e->line);
            case EK::Paren: {
                EOut in = gen_expr(g, e->l);
                in.code = "(" + in.code + ")";
                return in;
            }
            case EK::Local: {
                auto it = g.locals.find(e->var);
                if (it == g.locals.end()) fail("use of an undeclared local '" + e->var->name + "'", e->line);
                o.code = it->second.cname;
                o.type = it->second.type;
                o.tainted = it->second.tainted;
                o.arr_size = it->second.arr_size;
                o.arr_name = it->second.cname;
                return o;
            }
            case EK::Global:
            case EK::Upval: {
                const void *id;
                Value cur = current_value(g.fn, e, &id);
                auto m = mutables_.find(id);
                if (m != mutables_.end()) {
                    o.code = "c.mg[" + std::to_string(m->second) + "]";
                    o.tainted = true;
                    return o;
                }
                if (cur.is_number()) { o.code = num_literal(cur.num()); return o; }
                if (cur.is_boolean()) { o.code = cur.boolean_value() ? "true" : "false"; o.type = VT::Bool; return o; }
                if (cur.is_table()) return const_table(cur, e->line);
                fail("script-level variable '" + var_name(g.fn, e) + "' is " + State::type_name(cur) + " (only numbers, booleans and numeric tables can be used)", e->line);
            }
            case EK::Index: {
                Value sv;
                if (static_value(g.fn, e, &sv) && sv.is_number()) {  // math.pi, math.huge
                    o.code = num_literal(sv.num());
                    return o;
                }
                EOut t = gen_expr(g, e->l);
                if (t.type != VT::Arr) fail("only numeric arrays can be indexed", e->line);
                EOut k = gen_expr(g, e->r);
                if (k.type != VT::Num) fail("array index must be a number", e->line);
                o.code = t.arr_name + "[lt_idx(c, " + k.code + ", " + std::to_string(t.arr_size) + ")]";
                o.tainted = t.tainted;
                return o;
            }
            case EK::Call: {
                std::vector<EOut> res = gen_call(g, e, 1);
                if (res.empty()) fail("a function that returns nothing is used as a value", e->line);
                return res[0];
            }
            case EK::Add: case EK::Sub: case EK::Mul: case EK::Div: {
                EOut a = num_operand(g, e->l), b = num_operand(g, e->r);
                const char *op = e->k == EK::Add ? " + " : e->k == EK::Sub ? " - " : e->k == EK::Mul ? " * " : " / ";
                o.tainted = a.tainted || b.tainted;  // LtD operators propagate the error bound
                o.code = "(" + a.code + op + b.code + ")";
                return o;
            }
            case EK::Mod: {
                EOut a = num_operand(g, e->l), b = num_operand(g, e->r);
                o.tainted = a.tainted || b.tainted;
                o.code = std::string(o.tainted ? "lt_modD(c, " : "lt_mod(") + a.code + ", " + b.code + ")";
                return o;
            }
            case EK::Pow: {
                EOut a = num_operand(g, e->l), b = num_operand(g, e->r);
                o.code = "lt_pow(" + a.code + ", " + b.code + ")";
                o.tainted = true;
                return o;
            }
            case EK::Neg: {
                EOut a = num_operand(g, e->l);
                o.code = "(-" + a.code + ")";
                o.tainted = a.tainted;
                return o;
            }
            case EK::Len: {
                EOut a = gen_expr(g, e->l);
                if (a.type != VT::Arr) fail("'#' is only supported on numeric arrays", e->line);
                o.code = num_literal(a.arr_size);
                return o;
            }
            case EK::Not: {
                EOut a = gen_expr(g, e->l);
                if (a.type != VT::Bool) fail("'not' needs a boolean operand", e->line);
                o.code = "(!" + a.code + ")";
                o.type = VT::Bool;
                return o;
            }
            case EK::And: case EK::Or: {
                EOut a = gen_expr(g, e->l);
                // the right operand may only be evaluated when the left one does not decide
                const std::string saved = g.out.str();
                g.out.str("");
                ++g.indent;
                EOut b = gen_expr(g, e->r);
                --g.indent;
                const std::string pre = g.out.str();
                g.out.str(saved);
                g.out.seekp(0, std::ios::end);
                if (a.type != VT::Bool || b.type != VT::Bool) fail("'and'/'or' are only supported on booleans", e->line);
                o.type = VT::Bool;
                if (pre.empty()) {
                    o.code = "(" + a.code + (e->k == EK::And ? " && " : " || ") + b.code + ")";
                    return o;
                }
                std::string sc = new_tmp(g, "sc");
                line(g, "bool " + sc + " = " + a.code + ";");
                line(g, std::string("if (") + (e->k == EK::And ? "" : "!") + sc + ") {");
                g.out << pre;
                ++g.indent;
                line(g, sc + " = " + b.code + ";");
                --g.indent;
                line(g, "}");
                o.code = sc;
                return o;
            }
            case EK::Eq: case EK::Ne: case EK::Lt: case EK::Le: case EK::Gt: case EK::Ge: {
                if (e->l->k == EK::Nil || e->r->k == EK::Nil) fail("comparisons with nil are not supported", e->line);
                EOut a = gen_expr(g, e->l), b = gen_expr(g, e->r);
                o.type = VT::Bool;
                if (a.type == VT::Bool && b.type == VT::Bool && (e->k == EK::Eq || e->k == EK::Ne)) {
                    o.code = "(" + a.code + (e->k == EK::Eq ? " == " : " != ") + b.code + ")";
                    return o;
                }
                if (a.type != VT::Num || b.type != VT::Num) fail("comparison of non-numbers", e->line);
                const char *op = e->k == EK::Eq ? "==" : e->k == EK::Ne ? "!=" : e->k == EK::Lt ? "<" : e->k == EK::Le ? "<=" : e->k == EK::Gt ? ">" : ">=";
                if (a.tainted || b.tainted) {
                    // flags a tie within the error bounds, then compares the values
                    const char *fn = e->k == EK::Eq ? "lt_eq" : e->k == EK::Ne ? "lt_ne" : e->k == EK::Lt ? "lt_lt" : e->k == EK::Le ? "lt_le" : e->k == EK::Gt ? "lt_gt" : "lt_ge";
                    o.code = std::string(fn) + "(c, " + a.code + ", " + b.code + ")";
                } else {
                    o.code = "(" + a.code + " " + op + " " + b.code + ")";
                }
                return o;
            }
        }
        fail("unsupported expression", e->line);
    }

    EOut num_operand(Gen &g, const Expr *e) {
        EOut a = gen_expr(g, e);
        if (a.type != VT::Num) fail("arithmetic on a non-number", e->line);
        return a;
    }

    EOut const_table(const Value &tv, int line_no) {
        const Table *t = static_cast<const Table *>(tv.obj());
        auto it = table_names_.find(t);
        EOut o;
        o.type = VT::Arr;
        o.arr_size = static_cast<int>(t->arr.size());
        if (!t->hash.empty() || t->arr.empty()) fail("only plain numeric arrays can be used as tables", line_no);
        if (it == table_names_.end()) {
            std::string name = "lt_tab" + std::to_string(table_names_.size());
            tables_ << "LT_CONST double " << name << "[" << t->arr.size() + 1 << "] = {0.0";
            for (const Value &v : t->arr) {
                if (!v.is_number()) fail("only plain numeric arrays can be used as tables", line_no);
                tables_ << ", " << num_literal(v.num());
            }
            tables_ << "};\n";
            it = table_names_.emplace(t, name).first;
        }
        o.arr_name = it->second;
        o.code = it->second;
        return o;
    }

    // evaluates the argument list (last call expands) into single-value expressions
    std::vector<EOut> gen_args(Gen &g, const std::vector<Expr *> &list) {
        std::vector<EOut> args;
        for (size_t i = 0; i < list.size(); ++i) {
            const Expr *a = list[i];
            if (i + 1 == list.size() && a->k == EK::Call) {
                std::vector<EOut> many = gen_call(g, a, -1);
                for (EOut &m : many) args.push_back(m);
            } else {
                args.push_back(gen_expr(g, a));
            }
        }
        return args;
    }

    // want: number of results needed (-1 = all).  Emits the call as pre-statements.
    std::vector<EOut> gen_call(Gen &g, const Expr *e, int want) {
        Value callee;
        if (!static_value(g.fn, e->l, &callee) || !callee.is_function()) fail("cannot resolve the function being called", e->line);
        std::vector<EOut> res;
        auto bi = builtins_.find(callee.obj());
        if (bi != builtins_.end()) {
            const std::string &n = bi->second.name;
            std::vector<EOut> a = gen_args(g, e->list);
            for (EOut &x : a)
                if (x.type != VT::Num) fail("non-numeric argument to " + n, e->line);
            bool tin = false;
            for (EOut &x : a) tin = tin || x.tainted;
            auto need = [&](size_t k) {
                if (a.size() < k) fail("too few arguments to " + n, e->line);
            };
            auto one = [&](const std::string &code, bool tainted) {
                EOut o;
                o.code = code;
                o.tainted = tainted;
                res.push_back(o);
            };
            // the interpreter would print once per pixel; a silent device build would change the console output
            if (n == "print") fail("print() inside the " + scope_ + " function", e->line);
            if (n == "math.abs") { need(1); one(std::string(tin ? "lt_fabs(" : "fabs(") + a[0].code + ")", tin); return res; }
            if (n == "math.sqrt") { need(1); one(std::string(tin ? "lt_sqrt(" : "sqrt(") + a[0].code + ")", tin); return res; }
            if (n == "math.floor" || n == "math.ceil") {
                need(1);
                const bool fl = n == "math.floor";
                if (tin) one(std::string(fl ? "lt_floorD" : "lt_ceilD") + "(c, " + a[0].code + ")", false);  // exact once it is unambiguous
                else one(std::string(fl ? "floor(" : "ceil(") + a[0].code + ")", false);
                return res;
            }
            if (n == "math.fmod") {
                need(2);
                one(std::string(tin ? "lt_fmodD(c, " : "fmod(") + a[0].code + ", " + a[1].code + ")", tin);
                return res;
            }
            if (n == "math.deg") { need(1); one("(" + a[0].code + " / (LT_PI / 180.0))", tin); return res; }
            if (n == "math.rad") { need(1); one("(" + a[0].code + " * (LT_PI / 180.0))", tin); return res; }
            if (n == "math.max" || n == "math.min") {
                need(1);
                const bool mx = n == "math.max";
                std::string acc = a[0].code;
                for (size_t i = 1; i < a.size(); ++i) {
                    if (tin) acc = std::string(mx ? "lt_maxD(c, " : "lt_minD(c, ") + acc + ", " + a[i].code + ")";
                    else acc = std::string(mx ? "lt_max(" : "lt_min(") + acc + ", " + a[i].code + ")";
                }
                one(acc, tin);
                return res;
            }
            if (n == "math.log") {
                need(1);
                if (a.size() >= 2) one("lt_logb(" + a[0].code + ", " + a[1].code + ")", true);
                else one("lt_log(" + a[0].code + ")", true);
                return res;
            }
            if (n == "math.atan2" || n == "math.pow") {
                need(2);
                one(std::string(n == "math.atan2" ? "lt_atan2(" : "lt_pow(") + a[0].code + ", " + a[1].code + ")", true);
                return res;
            }
            if (n == "math.modf") {
                need(1);
                std::string t = new_tmp(g, "mf");
                if (tin) line(g, "LtD " + t + "[2]; lt_modfD(c, " + a[0].code + ", " + t + ");");
                else line(g, "double " + t + "[2]; lt_modf(" + a[0].code + ", " + t + ");");
                one(t + "[0]", tin);
                one(t + "[1]", tin);
                return res;
            }
            if (n == "latlon_to_ray") {
                need(2);
                std::string t = new_tmp(g, "lr");
                line(g, "double " + t + "[3]; lt_latlon_to_ray(c, " + a[0].code + ", " + a[1].code + ", " + t + ");");
                for (int i = 0; i < 3; ++i) one(t + "[" + std::to_string(i) + "]", false);
                return res;
            }
            if (n == "ray_to_latlon") {
                need(3);
                std::string t = new_tmp(g, "rl");
                line(g, "LtD " + t + "[2]; lt_ray_to_latlon(c, " + a[0].code + ", " + a[1].code + ", " + a[2].code + ", " + t + ");");
                for (int i = 0; i < 2; ++i) one(t + "[" + std::to_string(i) + "]", true);
                return res;
            }
            if (n == "plate_to_ray") {
                need(3);
                std::string t = new_tmp(g, "pr");
                line(g, "double " + t + "[3]; if (!lt_plate_to_ray(c, " + a[0].code + ", " + a[1].code + ", " + a[2].code + ", " + t + ")) { " +
                            (want == -2 ? std::string("return false;") : std::string("c.flag |= LT_RISK_NIL;")) + " }");
                for (int i = 0; i < 3; ++i) one(t + "[" + std::to_string(i) + "]", false);
                return res;
            }
            // plain one-argument libm functions
            static const char *kOne[] = {"acos", "asin", "atan", "cos", "cosh", "exp", "log10", "sin", "sinh", "tan", "tanh"};
            for (const char *f : kOne)
                if (n == std::string("math.") + f) {
                    need(1);
                    one(std::string("lt_") + f + "(" + a[0].code + ")", true);
                    return res;
                }
            fail("unsupported builtin " + n, e->line);
        }
        // ---- user function
        const Function *cf = static_cast<const Function *>(callee.obj());
        if (cf->cfn) fail("call to an unsupported C function", e->line);
        FuncInfo &fi = gen_function(cf);
        std::vector<EOut> a = gen_args(g, e->list);
        std::ostringstream callexpr;
        callexpr << fi.cname << "(c";
        for (int i = 0; i < cf->proto->nparams; ++i) {
            if (static_cast<size_t>(i) < a.size()) {
                if (a[static_cast<size_t>(i)].type != VT::Num) fail("non-numeric argument in a call to " + cf->proto->name, e->line);
                // an entry point (e.g. globe_plate called by the lens) takes exact doubles: an argument with an
                // error bound is accepted only when that bound is zero at run time
                if (fi.exact_params[static_cast<size_t>(i)] && a[static_cast<size_t>(i)].tainted)
                    callexpr << ", lt_exact(c, " << a[static_cast<size_t>(i)].code << ")";
                else
                    callexpr << ", " << a[static_cast<size_t>(i)].code;
            } else {
                callexpr << ", LT_NAN";  // missing argument = nil; using it would be an error in Lua too
            }
        }
        std::string t = new_tmp(g, "rv");
        callexpr << ", " << t << ")";
        line(g, "LtD " + t + "[" + std::to_string(std::max(1, fi.arity)) + "];");
        if (want == -2) {
            // `return f(...)`: a nil result of f is a nil result of ours
            line(g, "if (!" + callexpr.str() + ") return false;");
        } else {
            // used as a value: a nil here would be a Lua error; let the host look at this pixel
            line(g, "if (!" + callexpr.str() + ") c.flag |= LT_RISK_NIL;");
        }
        for (int i = 0; i < fi.arity; ++i) {
            EOut o;
            o.code = t + "[" + std::to_string(i) + "]";
            o.tainted = true;
            if (static_cast<size_t>(i) < fi.res_types.size() && fi.res_types[static_cast<size_t>(i)] == static_cast<int>(VT::Bool)) {
                o.code = "(" + o.code + ".v != 0.0)";
                o.type = VT::Bool;
                o.tainted = false;
            }
            res.push_back(o);
        }
        return res;
    }

    // results travel as LtD; a boolean result is 1.0 / 0.0 (exact) and is decoded at the call site
    std::string encode_result(Gen &g, size_t i, const EOut &v, int line_no) {
        if (v.type == VT::Arr) fail("arrays cannot be returned", line_no);
        if (g.fi->res_types.size() <= i) g.fi->res_types.resize(i + 1, -1);
        int &t = g.fi->res_types[i];
        if (t == -1) t = static_cast<int>(v.type);
        else if (t != static_cast<int>(v.type)) fail("a function returns a number on one path and a boolean on another", line_no);
        return v.type == VT::Bool ? "LtD(" + v.code + " ? 1.0 : 0.0)" : v.code;
    }

    // ------------------------------------------------------------------ statements
    void gen_block(Gen &g, const Block *b) {
        for (const Stmt *s : b->stmts) gen_stmt(g, s);
    }

    LocalInfo &declare(Gen &g, const VarInfo *v, VT type) {
        LocalInfo &li = g.locals[v];  // keeps the taint computed by the pre-pass
        li.cname = "v" + std::to_string(next_local_++) + "_" + sanitize(v->name);
        li.type = type;
        return li;
    }

    void gen_stmt(Gen &g, const Stmt *s) {
        switch (s->k) {
            case SK::Local: {
                if (s->vars.size() == 1 && s->exprs.size() == 1 && s->exprs[0]->k == EK::Table) {
                    const Expr *t = s->exprs[0];
                    if (!t->keys.empty()) fail("only positional numeric table constructors are supported", s->line);
                    std::vector<EOut> vals;
                    for (size_t i = 0; i < t->list.size(); ++i) {
                        const Expr *x = t->list[i];
                        if (x->k == EK::Call && i + 1 == t->list.size() && call_arity(g.fn, x) != 1)
                            fail("a multi-value call at the end of a table constructor is not supported", s->line);
                        vals.push_back(num_operand(g, x));
                    }
                    LocalInfo &li = declare(g, s->vars[0], VT::Arr);
                    li.arr_size = static_cast<int>(vals.size());
                    for (EOut &v : vals)
                        if (v.tainted && !li.tainted) fail("internal: array taint mismatch", s->line);
                    line(g, std::string(li.tainted ? "LtD " : "double ") + li.cname + "[" + std::to_string(vals.size() + 1) + "];");
                    line(g, li.cname + "[0] = 0.0;");
                    for (size_t i = 0; i < vals.size(); ++i) line(g, li.cname + "[" + std::to_string(i + 1) + "] = " + vals[i].code + ";");
                    return;
                }
                std::vector<EOut> vals = gen_args(g, s->exprs);
                // evaluate everything first (the new names become visible only afterwards)
                std::vector<std::string> tmps;
                for (size_t i = 0; i < s->vars.size() && i < vals.size(); ++i) {
                    std::string t = new_tmp(g, "in");
                    line(g, std::string(vals[i].type == VT::Bool ? "const bool " : vals[i].tainted ? "const LtD " : "const double ") + t + " = " + vals[i].code + ";");
                    tmps.push_back(t);
                }
                for (size_t i = 0; i < s->vars.size(); ++i) {
                    VT ty = i < vals.size() ? vals[i].type : VT::Num;
                    if (ty == VT::Arr) fail("arrays cannot be copied", s->line);
                    LocalInfo &li = declare(g, s->vars[i], ty);
                    if (i < vals.size() && vals[i].tainted && !li.tainted) fail("internal: taint mismatch", s->line);
                    line(g, std::string(ty == VT::Bool ? "bool " : li.tainted ? "LtD " : "double ") + li.cname + " = " + (i < tmps.size() ? tmps[i] : std::string("LT_NAN")) + ";");
                }
                return;
            }
            case SK::Assign: {
                std::vector<EOut> vals = gen_args(g, s->exprs);
                if (vals.size() < s->targets.size()) fail("assignment of nil is not supported", s->line);
                std::vector<std::string> tmps;
                for (size_t i = 0; i < s->targets.size(); ++i) {
                    std::string t = new_tmp(g, "as");
                    line(g, std::string(vals[i].type == VT::Bool ? "const bool " : vals[i].tainted ? "const LtD " : "const double ") + t + " = " + vals[i].code + ";");
                    tmps.push_back(t);
                }
                for (size_t i = s->targets.size(); i-- > 0;) {
                    const Expr *t = s->targets[i];
                    if (t->k == EK::Local) {
                        auto it = g.locals.find(t->var);
                        if (it == g.locals.end()) fail("assignment to an undeclared local", s->line);
                        if (it->second.type == VT::Arr) fail("arrays cannot be reassigned", s->line);
                        if ((it->second.type == VT::Bool) != (vals[i].type == VT::Bool)) fail("a variable changes type", s->line);
                        if (vals[i].tainted && !it->second.tainted) fail("internal: taint mismatch", s->line);
                        line(g, it->second.cname + " = " + tmps[i] + ";");
                    } else if (t->k == EK::Global || t->k == EK::Upval) {
                        const void *id;
                        current_value(g.fn, t, &id);
                        if (vals[i].type != VT::Num) fail("script-level variables assigned by the lens must be numbers", s->line);
                        line(g, "c.mg[" + std::to_string(mutables_.at(id)) + "] = " + tmps[i] + ";");
                    } else if (t->k == EK::Index) {
                        EOut arr = gen_expr(g, t->l);
                        if (arr.type != VT::Arr || t->l->k != EK::Local) fail("only local numeric arrays can be written", s->line);
                        EOut k = num_operand(g, t->r);
                        if (vals[i].tainted && !arr.tainted) fail("internal: array taint mismatch", s->line);
                        line(g, arr.arr_name + "[lt_idx(c, " + k.code + ", " + std::to_string(arr.arr_size) + ")] = " + tmps[i] + ";");
                    } else {
                        fail("unsupported assignment target", s->line);
                    }
                }
                return;
            }
            case SK::Call: {
                if (s->e->k != EK::Call) fail("unsupported call statement", s->line);
                gen_call(g, s->e, 0);
                return;
            }
            case SK::Do: {
                line(g, "{");
                ++g.indent;
                gen_block(g, s->body);
                --g.indent;
                line(g, "}");
                return;
            }
            case SK::While: {
                line(g, "for (;;) {");
                ++g.indent;
                EOut c = gen_expr(g, s->e);
                if (c.type != VT::Bool) fail("loop condition must be a boolean", s->line);
                line(g, "if (!" + c.code + ") break;");
                line(g, "if (++c.steps > LT_MAX_STEPS) { c.flag |= LT_RISK_LOOP; break; }");
                gen_block(g, s->body);
                --g.indent;
                line(g, "}");
                return;
            }
            case SK::Repeat: {
                line(g, "for (;;) {");
                ++g.indent;
                gen_block(g, s->body);
                EOut c = gen_expr(g, s->e);
                if (c.type != VT::Bool) fail("loop condition must be a boolean", s->line);
                line(g, "if (" + c.code + ") break;");
                line(g, "if (++c.steps > LT_MAX_STEPS) { c.flag |= LT_RISK_LOOP; break; }");
                --g.indent;
                line(g, "}");
                return;
            }
            case SK::If: {
                size_t opened = 0;
                for (size_t i = 0; i < s->conds.size(); ++i) {
                    EOut c = gen_expr(g, s->conds[i]);
                    if (c.type != VT::Bool) fail("'if' condition must be a boolean", s->line);
                    line(g, "if (" + c.code + ") {");
                    ++g.indent;
                    gen_block(g, s->blocks[i]);
                    --g.indent;
                    line(g, "} else {");
                    ++g.indent;
                    ++opened;
                }
                if (s->blocks.size() > s->conds.size()) gen_block(g, s->blocks.back());
                for (size_t i = 0; i < opened; ++i) {
                    --g.indent;
                    line(g, "}");
                }
                return;
            }
            case SK::NumFor: {
                EOut a = num_operand(g, s->exprs[0]), b = num_operand(g, s->exprs[1]);
                EOut st;
                st.code = "1.0";
                if (s->exprs.size() > 2) st = num_operand(g, s->exprs[2]);
                std::string i = new_tmp(g, "fi"), lim = new_tmp(g, "fl"), step = new_tmp(g, "fs");
                // loop bounds that depend on libm results: only accepted when they are exact at run time
                auto plain = [&](const EOut &v) { return v.tainted ? "lt_exact(c, " + v.code + ")" : v.code; };
                line(g, "const double " + lim + " = " + plain(b) + ", " + step + " = " + plain(st) + ";");
                line(g, "for (double " + i + " = " + plain(a) + "; " + step + " > 0 ? " + i + " <= " + lim + " : " + lim + " <= " + i + "; " + i + " = " + i + " + " + step + ") {");
                ++g.indent;
                line(g, "if (++c.steps > LT_MAX_STEPS) { c.flag |= LT_RISK_LOOP; break; }");
                LocalInfo &li = declare(g, s->vars[0], VT::Num);
                line(g, std::string(li.tainted ? "LtD " : "double ") + li.cname + " = " + i + ";");
                gen_block(g, s->body);
                --g.indent;
                line(g, "}");
                return;
            }
            case SK::Return: {
                const int K = g.fi->arity;
                if (s->exprs.empty() || (s->exprs.size() == 1 && s->exprs[0]->k == EK::Nil)) {
                    line(g, "return false;");
                    return;
                }
                // `return f(...)`: propagate f's nil
                if (s->exprs.size() == 1 && s->exprs[0]->k == EK::Call) {
                    std::vector<EOut> vals = gen_call(g, s->exprs[0], -2);
                    if (static_cast<int>(vals.size()) < K) fail("a function returns a different number of values on different paths", s->line);
                    for (int i = 0; i < K; ++i)
                        line(g, "r[" + std::to_string(i) + "] = " + encode_result(g, static_cast<size_t>(i), vals[static_cast<size_t>(i)], s->line) + ";");
                    line(g, "return true;");
                    return;
                }
                std::vector<EOut> vals = gen_args(g, s->exprs);
                if (static_cast<int>(vals.size()) != K) fail("a function returns a different number of values on different paths", s->line);
                std::vector<std::string> tmps;
                for (int i = 0; i < K; ++i) {
                    std::string t = new_tmp(g, "re");
                    line(g, "const LtD " + t + " = " + encode_result(g, static_cast<size_t>(i), vals[static_cast<size_t>(i)], s->line) + ";");
                    tmps.push_back(t);
                }
                for (int i = 0; i < K; ++i) line(g, "r[" + std::to_string(i) + "] = " + tmps[static_cast<size_t>(i)] + ";");
                line(g, "return true;");
                return;
            }
            case SK::Break: line(g, "break;"); return;
            case SK::GenFor: fail("generic 'for ... in' is not supported", s->line);
            case SK::LocalFunction: fail("local functions inside the lens are not supported", s->line);
            case SK::Goto:
            case SK::Label: fail("goto is not supported", s->line);
        }
    }

    State &L_;
    std::map<const Object *, BuiltinInfo> builtins_;
    std::map<const void *, int> mutables_;
    std::vector<double> mutable_init_;
    std::map<const Function *, FuncInfo> funcs_;
    std::vector<std::string> order_;
    std::ostringstream tables_;
    std::map<const Table *, std::string> table_names_;
    std::set<const Function *> entry_fns_;  // their parameters are exact doubles
    std::string scope_ = "lens";            // names the function being translated in error messages
    int next_local_ = 0;
};

}  // namespace

TranspileResult transpile_lens(State &L, const Value &lens_inverse, const Value *globe_plate) {
    Transpiler t(L);
    return t.run(&lens_inverse, 2, 3, "lens_inverse", globe_plate);
}

TranspileResult transpile_lens_forward(State &L, const Value &lens_forward, const Value *globe_plate) {
    Transpiler t(L);
    return t.run(&lens_forward, 3, 2, "lens_forward", globe_plate);
}

TranspileResult transpile_globe_plate(State &L, const Value &globe_plate) {
    Transpiler t(L);
    return t.run(nullptr, 0, 0, "globe_plate", &globe_plate);
}

std::string transpile_prelude(bool cuda, bool noinline_user_functions) {
    std::string s;
    if (cuda) {
        s += "#define LT_FN static __device__ __forceinline__\n#define LT_HD __device__ __forceinline__\n#define LT_CONST static __device__ const\n";
        // translated script functions: inlined by default; real calls cut NVRTC's time on big lenses
        // (quincuncial 1.2 s -> 0.5 s) at some cost in the kernel
        s += noinline_user_functions ? "#define LT_UFN static __device__ __noinline__\n" : "#define LT_UFN static __device__ __forceinline__\n";
        s += "#define LT_NAN (__longlong_as_double(0x7ff8000000000000LL))\n#define LT_INF (__longlong_as_double(0x7ff0000000000000LL))\n";
    } else {
        s += "#include <math.h>\n#define LT_FN static inline\n#define LT_UFN static\n#define LT_HD inline\n#define LT_CONST static const\n";
        s += "#define LT_NAN (__builtin_nan(\"\"))\n#define LT_INF (__builtin_inf())\n";
    }
    s += R"PRE(
#define LT_PI 3.14159265358979323846
#define LT_MAX_STEPS 100000
#define LT_RISK_NEAR 1u     /* a comparison / rounding decision lies within the error bound of its operands */
#define LT_RISK_NIL 2u      /* a nil showed up where the script uses a number (Lua would raise an error) */
#define LT_RISK_LOOP 4u     /* runaway loop */
#define LT_RISK_INDEX 8u    /* array index out of range / not an integer */
#define LT_RISK_F32 32u     /* a value sits on a float32 rounding boundary */
#define LT_MAX_MUT 32

/* A double that went through a libm function, with a bound `e` on |value computed here - value the
 * host's libm would give| that holds to all orders: every rule below bounds the change of its function
 * over the whole input interval [v - e, v + e] (box, for two operands), and gives an infinite bound
 * when that interval reaches a pole, a domain edge or a NaN region.  e == 0: provably identical. */
struct LtD {
    double v, e;
    LT_HD LtD() {}
    LT_HD LtD(double x) : v(x), e(0.0) {}
    LT_HD LtD(double x, double err) : v(x), e(err) {}
};
#define LT_U 0x1p-52            /* one rounding */
#define LT_KU (8.0 * LT_U)      /* libm results: CUDA <= 2 ulp + glibc <= 2 ulp (documented), doubled */
#define LT_FINITE(x) (fabs(x) <= 1.79769313486231570815e308)

struct LtPlate { float forward[3], right[3], up[3]; float dist; };

struct Ctx {
    unsigned flag;
    unsigned steps;
    LtD mg[LT_MAX_MUT];     /* script-level variables the lens assigns (per pixel copy) */
    const LtPlate *plates;
    int numplates;
};

/* result r of an IEEE operation whose inputs carried errors: propagated part + one rounding */
LT_FN LtD lt_mk(double r, double prop) { return LtD(r, !(prop == 0.0) ? prop + LT_U * fabs(r) : 0.0); }
/* result r of a libm function */
LT_FN LtD lt_fn(double r, double prop) {
    /* identical inputs and a NaN / infinite result (domain error, overflow): the same on both sides */
    if (prop == 0.0 && !(fabs(r) <= 1.79769313486231570815e308)) return LtD(r);
    return LtD(r, prop + LT_KU * fabs(r));
}
/* result r of exp, sinh, cosh, pow or atan2, whose finite arguments can put it at a range edge where LT_KU * |r|
 * says nothing: within a few ulp of the overflow threshold one libm may give the largest double and the other inf,
 * and below the normal range (an ulp is 2^-1074 there) one may give 0 and the other a subnormal.  edge: the
 * arguments are finite and not ones that make the result exact (sinh(0), pow(0, y), atan2(0, x), ...) */
LT_FN LtD lt_fn_edge(double r, double prop, bool edge) {
    if (edge && fabs(r) < 0x1p-1022) return LtD(r, prop + LT_KU * 0x1p-1022);
    if (edge && fabs(r) > 0x1.ffffffffffff0p1023) return LtD(r, LT_INF);
    return lt_fn(r, prop);
}
/* exp(e) - 1 <= e / (1 - e) for 0 <= e < 1: the relative change of exp over [v - e, v + e] */
LT_FN double lt_expm1_bound(double e) { return e < 1.0 ? e / (1.0 - e) : LT_INF; }

LT_FN LtD operator+(LtD a, LtD b) { return lt_mk(a.v + b.v, a.e + b.e); }
LT_FN LtD operator-(LtD a, LtD b) { return lt_mk(a.v - b.v, a.e + b.e); }
LT_FN LtD operator*(LtD a, LtD b) {
    const double r = a.v * b.v;
    if (a.e == 0.0 && b.e == 0.0) return LtD(r);
    return lt_mk(r, fabs(a.v) * b.e + fabs(b.v) * a.e + a.e * b.e);
}
LT_FN LtD operator/(LtD a, LtD b) {
    const double r = a.v / b.v;
    if (a.e == 0.0 && b.e == 0.0) return LtD(r);
    /* |a'/b' - a/b| <= (a.e + |a/b| b.e) / (|b| - b.e); unbounded once the divisor's interval reaches 0 */
    const double d = fabs(b.v) - b.e;
    return lt_mk(r, d > 0.0 ? (a.e + fabs(r) * b.e) / d : LT_INF);
}
LT_FN LtD operator-(LtD a) { return LtD(-a.v, a.e); }
LT_FN LtD lt_fabs(LtD a) { return LtD(fabs(a.v), a.e); }
LT_FN LtD lt_sqrt(LtD a) {
    const double r = sqrt(a.v);
    if (a.e == 0.0) return LtD(r);
    /* sqrt(v) - sqrt(v - e) = e / (r + sqrt(v - e)) <= e / (2r - e/r), as sqrt(1 - t) >= 1 - t; NaN below 0 */
    return lt_mk(r, a.e < a.v ? a.e / (2.0 * r - a.e / r) : LT_INF);
}
LT_FN LtD lt_sin(LtD a) { return lt_fn(sin(a.v), a.e); }
LT_FN LtD lt_cos(LtD a) { return lt_fn(cos(a.v), a.e); }
LT_FN LtD lt_tan(LtD a) {
    const double r = tan(a.v);
    if (a.e == 0.0) return lt_fn(r, 0.0);
    /* tan(v + s) - tan(v) = (1 + r^2) tan(s) / (1 - r tan(s)), and tan(s) <= s / (1 - s^2/2) for s < sqrt(2);
     * the denominator reaching 0 means the interval reaches a pole */
    const double t = a.e * a.e < 2.0 ? a.e / (1.0 - 0.5 * a.e * a.e) : LT_INF;
    const double d = 1.0 - fabs(r) * t;
    return lt_fn(r, d > 0.0 ? (1.0 + r * r) * t / d : LT_INF);
}
/* asin, acos: the derivative at the end of the interval nearer +-1; NaN beyond */
LT_FN double lt_asin_bound(LtD a) {
    const double m = fabs(a.v) + a.e;
    return a.e == 0.0 ? 0.0 : m < 1.0 ? a.e / sqrt((1.0 - m) * (1.0 + m)) : LT_INF;
}
LT_FN LtD lt_asin(LtD a) { return lt_fn(asin(a.v), lt_asin_bound(a)); }
LT_FN LtD lt_acos(LtD a) { return lt_fn(acos(a.v), lt_asin_bound(a)); }
LT_FN LtD lt_atan(LtD a) {
    const double m = fmax(fabs(a.v) - a.e, 0.0);   /* the derivative at the end of the interval nearer 0 */
    return lt_fn(atan(a.v), a.e / (1.0 + m * m));
}
LT_FN LtD lt_atan2(LtD y, LtD x) {
    const double r = atan2(y.v, x.v);
    const bool edge = y.v != 0.0 && LT_FINITE(y.v) && LT_FINITE(x.v);   /* atan2(tiny, huge) underflows */
    if (y.e == 0.0 && x.e == 0.0) return lt_fn_edge(r, 0.0, edge);
    /* along a path inside the error box, |d atan2| = |x dy - y dx| / (x^2 + y^2), the box's nearest point to the
     * origin bounding the denominator; a box holding the origin, or one that can move y across 0 where x < 0
     * (atan2 jumps by 2 pi there), has no bound */
    const double dy = fmax(fabs(y.v) - y.e, 0.0), dx = fmax(fabs(x.v) - x.e, 0.0);
    const bool jump = dy == 0.0 && (dx == 0.0 || (y.e > 0.0 && x.v - x.e < 0.0));
    return lt_fn_edge(r, jump ? LT_INF : (fabs(x.v) * y.e + fabs(y.v) * x.e + 2.0 * x.e * y.e) / (dx * dx + dy * dy), edge);
}
LT_FN LtD lt_exp(LtD a) {
    const double r = exp(a.v);
    return lt_fn_edge(r, a.e == 0.0 ? 0.0 : r * lt_expm1_bound(a.e), LT_FINITE(a.v));
}
/* log(v) - log(v - e) = -log(1 - t) <= t / (1 - t), t = e / v; unbounded once the interval reaches 0 */
LT_FN double lt_log_bound(LtD a) {
    const double t = a.e / fabs(a.v);
    return a.e == 0.0 ? 0.0 : t < 1.0 ? t / (1.0 - t) : LT_INF;
}
LT_FN LtD lt_log(LtD a) { return lt_fn(log(a.v), lt_log_bound(a)); }
LT_FN LtD lt_log10(LtD a) { return lt_fn(log10(a.v), lt_log_bound(a) / 2.302585092994046); }
LT_FN LtD lt_logb(LtD x, LtD base) {   /* lmathlib.c math_log with a base */
    if (base.e == 0.0 && base.v == 10.0) return lt_log10(x);
    return lt_log(x) / lt_log(base);
}
/* sinh(v + s) - sinh(v) = sinh(v) (cosh(s) - 1) + cosh(v) sinh(s), cosh(v) <= |r| + 1: at most (|r| + 1) (exp(e) - 1) */
LT_FN LtD lt_sinh(LtD a) {
    const double r = sinh(a.v);
    return lt_fn_edge(r, a.e == 0.0 ? 0.0 : (fabs(r) + 1.0) * lt_expm1_bound(a.e), a.v != 0.0 && LT_FINITE(a.v));
}
LT_FN LtD lt_cosh(LtD a) {
    const double r = cosh(a.v);
    return lt_fn_edge(r, a.e == 0.0 ? 0.0 : r * lt_expm1_bound(a.e), LT_FINITE(a.v));
}
LT_FN LtD lt_tanh(LtD a) { return lt_fn(tanh(a.v), a.e); }
LT_FN LtD lt_pow(LtD a, LtD b) {
    const double r = pow(a.v, b.v);
    const bool edge = a.v != 0.0 && LT_FINITE(a.v) && LT_FINITE(b.v);
    if (a.e == 0.0 && b.e == 0.0) return lt_fn_edge(r, 0.0, edge);
    const bool int_b = b.e == 0.0 && b.v == floor(b.v);
    if (a.v == 0.0)   /* |a'^b| <= a.e^b for a positive exponent; a negative base gives NaN unless b is an integer */
        return lt_fn(r, b.e == 0.0 && b.v > 0.0 && int_b ? pow(a.e, b.v) : LT_INF);
    /* a'^b' = r exp(b (log a' - log a) + (b' - b) log a'), |log a' - log a| <= l = t / (1 - t), t = a.e / |a|: the
     * base keeps its sign (only an integer exponent is defined for a negative one), then |exp(w) - 1| <= z / (1 - z) */
    const double t = a.e / fabs(a.v);
    if (!(t < 1.0) || (b.e != 0.0 && !(a.v > 0.0))) return lt_fn(r, LT_INF);
    const double l = t / (1.0 - t);
    const double z = fabs(b.v) * l + (b.e == 0.0 ? 0.0 : b.e * (fabs(log(a.v)) + l));
    return lt_fn_edge(r, fabs(r) * lt_expm1_bound(z), edge);
}

/* ---- decisions: flag when the outcome is not certain within the bounds (x2 safety) ---- */
LT_FN void lt_tie(Ctx &c, LtD a, LtD b) {
    const double bound = 2.0 * (a.e + b.e);
    if (!(bound == 0.0) && !(fabs(a.v - b.v) > bound)) c.flag |= LT_RISK_NEAR;   /* also NaN / inf bounds */
}
LT_FN bool lt_lt(Ctx &c, LtD a, LtD b) { lt_tie(c, a, b); return a.v < b.v; }
LT_FN bool lt_le(Ctx &c, LtD a, LtD b) { lt_tie(c, a, b); return a.v <= b.v; }
LT_FN bool lt_gt(Ctx &c, LtD a, LtD b) { lt_tie(c, a, b); return a.v > b.v; }
LT_FN bool lt_ge(Ctx &c, LtD a, LtD b) { lt_tie(c, a, b); return a.v >= b.v; }
LT_FN bool lt_eq(Ctx &c, LtD a, LtD b) { lt_tie(c, a, b); return a.v == b.v; }
LT_FN bool lt_ne(Ctx &c, LtD a, LtD b) { lt_tie(c, a, b); return a.v != b.v; }
LT_FN double lt_max(double a, double b) { return b > a ? b : a; }  /* lmathlib.c math_max */
LT_FN double lt_min(double a, double b) { return b < a ? b : a; }
LT_FN LtD lt_maxD(Ctx &c, LtD a, LtD b) { lt_tie(c, a, b); return b.v > a.v ? b : a; }
LT_FN LtD lt_minD(Ctx &c, LtD a, LtD b) { lt_tie(c, a, b); return b.v < a.v ? b : a; }
LT_FN double lt_exact(Ctx &c, LtD a) { if (!(a.e == 0.0)) c.flag |= LT_RISK_NEAR; return a.v; }
LT_FN double lt_floorD(Ctx &c, LtD x) {
    const double f = floor(x.v);
    if (!(x.e == 0.0)) { lt_tie(c, x, LtD(f)); lt_tie(c, x, LtD(f + 1.0)); }
    return f;
}
LT_FN double lt_ceilD(Ctx &c, LtD x) {
    const double f = ceil(x.v);
    if (!(x.e == 0.0)) { lt_tie(c, x, LtD(f)); lt_tie(c, x, LtD(f - 1.0)); }
    return f;
}
LT_FN double lt_mod(double a, double b) { return a - floor(a / b) * b; }   /* luai_nummod */
LT_FN LtD lt_modD(Ctx &c, LtD a, LtD b) { return a - LtD(lt_floorD(c, a / b)) * b; }
LT_FN LtD lt_fmodD(Ctx &c, LtD a, LtD b) {
    const LtD q = a / b;
    const double t = trunc(q.v);
    if (!(q.e == 0.0)) { lt_tie(c, q, LtD(t)); lt_tie(c, q, LtD(t + (q.v < 0 ? -1.0 : 1.0))); }
    return LtD(fmod(a.v, b.v), a.e + fabs(t) * b.e);
}
LT_FN void lt_modf(double x, double *out) { double ip; out[1] = modf(x, &ip); out[0] = ip; }
LT_FN void lt_modfD(Ctx &c, LtD x, LtD *out) {
    double ip;
    const double fp = modf(x.v, &ip);
    if (!(x.e == 0.0)) { lt_tie(c, x, LtD(ip)); lt_tie(c, x, LtD(ip + (x.v < 0 ? -1.0 : 1.0))); }
    out[0] = LtD(ip);
    out[1] = LtD(fp, x.e);
}
LT_FN int lt_idx(Ctx &c, LtD k, int n) {
    const double f = floor(k.v);
    if (!(k.e == 0.0) || !(k.v == f) || !(k.v >= 1.0) || !(k.v <= (double)n)) { c.flag |= LT_RISK_INDEX; return 0; }
    return (int)f;
}
/* double -> float32 narrowing: certain only if the whole error interval rounds the same way */
LT_FN float lt_f32(Ctx &c, LtD x) {
    const float f = (float)x.v;
    if (!(x.e == 0.0)) {
        const double b = 2.0 * x.e;
        if ((float)(x.v - b) != f || (float)(x.v + b) != f) c.flag |= LT_RISK_F32;
    }
    return f;
}
/* CtoLUA_latlon_to_ray (fisheye.c:1494-1504): through a float32 vec3_t, hence exact again */
LT_FN void lt_latlon_to_ray(Ctx &c, LtD lat, LtD lon, double *out) {
    const LtD clat = lt_cos(lat);
    out[0] = (double)lt_f32(c, lt_sin(lon) * clat);
    out[1] = (double)lt_f32(c, lt_sin(lat));
    out[2] = (double)lt_f32(c, lt_cos(lon) * clat);
}
/* CtoLUA_ray_to_latlon (fisheye.c:1506-1519): arguments narrowed to float first */
LT_FN void lt_ray_to_latlon(Ctx &c, LtD rx, LtD ry, LtD rz, LtD *out) {
    const float x = lt_f32(c, rx), y = lt_f32(c, ry), z = lt_f32(c, rz);
    const float h2 = x * x + z * z;
    out[1] = lt_fn(atan2((double)x, (double)z), 0.0);
    out[0] = lt_fn(atan2((double)y, sqrt((double)h2)), 0.0);
}
/* CtoLUA_plate_to_ray (fisheye.c:1521-1537) + plate_uv_to_ray (:1198-1214) */
LT_FN bool lt_plate_to_ray(Ctx &c, LtD plate, LtD ud, LtD vd, double *out) {
    if (!(plate.e == 0.0)) { lt_tie(c, plate, LtD(trunc(plate.v))); lt_tie(c, plate, LtD(trunc(plate.v) + (plate.v < 0 ? -1.0 : 1.0))); }
    const int p = (int)plate.v;
    if (p < 0 || p >= c.numplates) return false;
    const LtPlate &P = c.plates[p];
    const LtD u = ud - LtD(0.5), v = -(vd - LtD(0.5));
    float r[3] = {0.0f, 0.0f, 0.0f};
    const float fu = lt_f32(c, u), fv = lt_f32(c, v);
    for (int i = 0; i < 3; ++i) r[i] = r[i] + P.dist * P.forward[i];
    for (int i = 0; i < 3; ++i) r[i] = r[i] + fu * P.right[i];
    for (int i = 0; i < 3; ++i) r[i] = r[i] + fv * P.up[i];
    float len = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    len = (float)sqrt((double)len);
    if (len) { const float inv = 1 / len; r[0] *= inv; r[1] *= inv; r[2] *= inv; }
    out[0] = (double)r[0]; out[1] = (double)r[1]; out[2] = (double)r[2];
    return true;
}
)PRE";
    return s;
}

}  // namespace blinky
