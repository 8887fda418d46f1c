// regex_compiler.cpp -- see regex_compiler.h.  Pure host C++ (no CUDA, no torch).
#include "regex_compiler.h"

#include <string.h>

#include <algorithm>
#include <map>
#include <set>
#include <stdexcept>

namespace lcb200 {
namespace {

// ------------------------------------------------------------------------------------------ byte sets
struct ByteSet {
    uint64_t w[4] = {0, 0, 0, 0};
    void set(unsigned b) { w[b >> 6] |= 1ull << (b & 63); }
    void set_range(unsigned lo, unsigned hi) {
        for (unsigned b = lo; b <= hi; ++b)
            set(b);
    }
    bool test(unsigned b) const { return (w[b >> 6] >> (b & 63)) & 1; }
    void invert() {
        for (auto& x : w)
            x = ~x;
    }
    void merge(const ByteSet& o) {
        for (int i = 0; i < 4; ++i)
            w[i] |= o.w[i];
    }
    bool empty() const { return !(w[0] | w[1] | w[2] | w[3]); }
    bool operator<(const ByteSet& o) const { return memcmp(w, o.w, sizeof w) < 0; }
    bool operator==(const ByteSet& o) const { return memcmp(w, o.w, sizeof w) == 0; }
};

// C-locale classes on `char` (SURVEY.md A.1): bytes >= 0x80 belong to none of them.
ByteSet cls_digit() {
    ByteSet s;
    s.set_range('0', '9');
    return s;
}
ByteSet cls_lower() {
    ByteSet s;
    s.set_range('a', 'z');
    return s;
}
ByteSet cls_upper() {
    ByteSet s;
    s.set_range('A', 'Z');
    return s;
}
ByteSet cls_alpha() {
    ByteSet s = cls_lower();
    s.merge(cls_upper());
    return s;
}
ByteSet cls_alnum() {
    ByteSet s = cls_alpha();
    s.merge(cls_digit());
    return s;
}
ByteSet cls_word() {
    ByteSet s = cls_alnum();
    s.set('_');
    return s;
}
ByteSet cls_space() {
    ByteSet s;
    s.set(' ');
    s.set_range('\t', '\r'); // \t \n \v \f \r
    return s;
}
ByteSet cls_blank() {
    ByteSet s;
    s.set(' ');
    s.set('\t');
    return s;
}
ByteSet cls_vspace() {
    ByteSet s;
    s.set_range('\n', '\r'); // \n \v \f \r
    return s;
}
ByteSet cls_cntrl() {
    ByteSet s;
    s.set_range(0, 31);
    s.set(127);
    return s;
}
ByteSet cls_print() {
    ByteSet s;
    s.set_range(32, 126);
    return s;
}
ByteSet cls_graph() {
    ByteSet s;
    s.set_range(33, 126);
    return s;
}
ByteSet cls_punct() {
    ByteSet s = cls_graph();
    ByteSet a = cls_alnum();
    for (int i = 0; i < 4; ++i)
        s.w[i] &= ~a.w[i];
    return s;
}
ByteSet cls_xdigit() {
    ByteSet s = cls_digit();
    s.set_range('a', 'f');
    s.set_range('A', 'F');
    return s;
}
ByteSet negate(ByteSet s) {
    s.invert();
    return s;
}

// ------------------------------------------------------------------------------------------ AST
enum AssertKind : uint32_t {
    A_BOL = 1u << 0,   // ^   (line start; boost default is multi-line)
    A_EOL = 1u << 1,   // $
    A_BOT = 1u << 2,   // \A \`
    A_EOT = 1u << 3,   // \z \'
    A_WORDB = 1u << 4, // \b
    A_NWORDB = 1u << 5, // \B
    A_WSTART = 1u << 6, // \<  (boost match_word_start: the next byte is a word byte, the previous one is not / absent)
    A_WEND = 1u << 7,   // \>  (boost match_word_end: the previous byte is a word byte, the next one is not / absent)
    A_LA0 = 1u << 8,    // bits 8..15: single-byte look-ahead i, (?=[set]) or (?![set]) -- Parser::las[i]
};
constexpr int kMaxLookAheads = 8;

enum NodeKind { N_EMPTY, N_SET, N_CAT, N_ALT, N_REP, N_GROUP, N_ASSERT };

struct Node {
    NodeKind kind = N_EMPTY;
    ByteSet set;
    std::vector<int> kids;
    int min = 0, max = 0; // max < 0 == unbounded
    bool greedy = true;
    int cap = -1; // capture index (1-based) or -1
    uint32_t akind = 0;
};

struct Unsupported : std::runtime_error {
    using std::runtime_error::runtime_error;
};
struct Invalid : std::runtime_error {
    using std::runtime_error::runtime_error;
};

struct LookAhead {
    ByteSet set;
    bool neg;
};

struct Parser {
    const unsigned char* p;
    size_t n, i = 0;
    std::vector<Node> nodes;
    std::vector<LookAhead> las; // (?=x) / (?!x) with a one-byte body: assertions on the NEXT byte
    int ncap = 0;
    bool icase = false;

    Parser(const char* s, size_t len) : p((const unsigned char*)s), n(len) {}

    int mk(NodeKind k) {
        nodes.emplace_back();
        nodes.back().kind = k;
        return (int)nodes.size() - 1;
    }
    bool more() const { return i < n; }
    int peek() const { return i < n ? p[i] : -1; }

    int mk_set(ByteSet s) {
        if (icase) {
            for (unsigned c = 'a'; c <= 'z'; ++c) {
                if (s.test(c) || s.test(c - 32)) {
                    s.set(c);
                    s.set(c - 32);
                }
            }
        }
        int id = mk(N_SET);
        nodes[id].set = s;
        return id;
    }
    int mk_byte(unsigned b) {
        ByteSet s;
        s.set(b);
        return mk_set(s);
    }

    int parse_alt() {
        std::vector<int> alts;
        alts.push_back(parse_cat());
        while (peek() == '|') {
            ++i;
            alts.push_back(parse_cat());
        }
        if (alts.size() == 1)
            return alts[0];
        int id = mk(N_ALT);
        nodes[id].kids = alts;
        return id;
    }

    int parse_cat() {
        std::vector<int> items;
        while (more() && peek() != '|' && peek() != ')') {
            int a = parse_repeat();
            if (a >= 0)
                items.push_back(a);
        }
        if (items.empty())
            return mk(N_EMPTY);
        if (items.size() == 1)
            return items[0];
        int id = mk(N_CAT);
        nodes[id].kids = items;
        return id;
    }

    static bool is_digit(int c) { return c >= '0' && c <= '9'; }

    // returns -1 for constructs that produce nothing (comments, flag groups)
    int parse_repeat() {
        bool is_atom = true;
        int a = parse_atom(is_atom);
        if (a < 0)
            return a;
        while (more()) {
            int c = peek();
            int mn, mx;
            if (c == '*') {
                mn = 0;
                mx = -1;
                ++i;
            } else if (c == '+') {
                mn = 1;
                mx = -1;
                ++i;
            } else if (c == '?') {
                mn = 0;
                mx = 1;
                ++i;
            } else if (c == '{') {
                size_t save = i;
                ++i;
                while (peek() == ' ')
                    ++i;
                if (!is_digit(peek()))
                    throw Invalid("invalid content of repeat range");
                long a1 = 0;
                while (is_digit(peek())) {
                    a1 = a1 * 10 + (p[i++] - '0');
                    if (a1 > 100000)
                        throw Unsupported("repeat count too large");
                }
                long a2 = a1;
                while (peek() == ' ')
                    ++i;
                if (peek() == ',') {
                    ++i;
                    while (peek() == ' ')
                        ++i;
                    if (is_digit(peek())) {
                        a2 = 0;
                        while (is_digit(peek())) {
                            a2 = a2 * 10 + (p[i++] - '0');
                            if (a2 > 100000)
                                throw Unsupported("repeat count too large");
                        }
                    } else {
                        a2 = -1;
                    }
                    while (peek() == ' ')
                        ++i;
                }
                if (peek() != '}')
                    throw Invalid("invalid content of repeat range");
                ++i;
                (void)save;
                if (a2 >= 0 && a2 < a1)
                    throw Invalid("repeat range min > max");
                mn = (int)a1;
                mx = (int)a2;
            } else {
                break;
            }
            if (!is_atom)
                throw Invalid("nothing to repeat");
            bool greedy = true;
            if (peek() == '?') {
                greedy = false;
                ++i;
            } else if (peek() == '+') {
                throw Unsupported("possessive quantifier");
            }
            int r = mk(N_REP);
            nodes[r].kids = {a};
            nodes[r].min = mn;
            nodes[r].max = mx;
            nodes[r].greedy = greedy;
            a = r;
            // a further quantifier directly applied to a quantifier ("a**") is rejected
            int c2 = peek();
            if (c2 == '*' || c2 == '+' || c2 == '?' || c2 == '{')
                throw Unsupported("stacked quantifiers");
        }
        return a;
    }

    int parse_group() {
        // at '('
        ++i;
        int cap = -1;
        bool saved_icase = icase;
        if (peek() == '?') {
            ++i;
            int c = peek();
            if (c == ':') {
                ++i;
            } else if (c == '#') {
                while (more() && peek() != ')')
                    ++i;
                if (!more())
                    throw Invalid("unterminated comment");
                ++i;
                return -1;
            } else if (c == '<' || c == '\'') {
                int close = c == '<' ? '>' : '\'';
                if (i + 1 < n && (p[i + 1] == '=' || p[i + 1] == '!'))
                    throw Unsupported("look-behind assertion");
                ++i;
                size_t s = i;
                while (more() && peek() != close)
                    ++i;
                if (!more() || i == s)
                    throw Invalid("bad group name");
                ++i;
                cap = ++ncap;
            } else if (c == '=' || c == '!') {
                // look-ahead whose body is exactly one byte (a literal, an escape, a class, '.'): an assertion on the
                // next byte, like $ and \b.  Anything longer would need the automaton to run ahead of itself.
                ++i;
                if (peek() == ')')
                    throw Unsupported("empty look-ahead");
                const int body = parse_alt();
                if (!more() || peek() != ')')
                    throw Invalid("unterminated look-ahead");
                ++i;
                icase = saved_icase;
                if (body < 0 || nodes[body].kind != N_SET)
                    throw Unsupported("look-ahead of more than one byte");
                if ((int)las.size() >= kMaxLookAheads)
                    throw Unsupported("more than 8 look-ahead assertions");
                las.push_back({nodes[body].set, c == '!'});
                int id = (int)nodes.size();
                nodes.push_back(Node());
                nodes[id].kind = N_ASSERT;
                nodes[id].akind = A_LA0 << (las.size() - 1);
                return id;
            } else if (c == '>') {
                throw Unsupported("atomic group");
            } else if (c == 'P') {
                throw Invalid("(?P is not boost syntax");
            } else {
                // inline flags: (?i) (?-i) (?i:...) ; s and m only in their default (on) state
                bool neg = false, any = false;
                bool new_icase = icase;
                while (more()) {
                    c = peek();
                    if (c == '-') {
                        neg = true;
                        ++i;
                    } else if (c == 'i') {
                        new_icase = !neg;
                        any = true;
                        ++i;
                    } else if (c == 's' || c == 'm') {
                        if (neg)
                            throw Unsupported("(?-s) / (?-m)");
                        any = true;
                        ++i;
                    } else if (c == 'x') {
                        throw Unsupported("(?x)");
                    } else {
                        break;
                    }
                }
                if (!any)
                    throw Unsupported("unsupported (? construct");
                if (peek() == ')') {
                    ++i;
                    icase = new_icase; // applies to the rest of the enclosing group
                    return -1;
                }
                if (peek() != ':')
                    throw Invalid("bad inline flags");
                ++i;
                icase = new_icase;
            }
        } else {
            cap = ++ncap;
        }
        int inner = parse_alt();
        if (peek() != ')')
            throw Invalid("missing )");
        ++i;
        icase = saved_icase;
        int g = mk(N_GROUP);
        nodes[g].kids = {inner};
        nodes[g].cap = cap;
        return g;
    }

    static int hexval(int c) {
        if (c >= '0' && c <= '9')
            return c - '0';
        if (c >= 'a' && c <= 'f')
            return c - 'a' + 10;
        if (c >= 'A' && c <= 'F')
            return c - 'A' + 10;
        return -1;
    }

    // class escapes shared by atom and set context; returns true if c named a class
    static bool class_escape(int c, ByteSet& out) {
        switch (c) {
            case 'd':
                out = cls_digit();
                return true;
            case 'D':
                out = negate(cls_digit());
                return true;
            case 'w':
                out = cls_word();
                return true;
            case 'W':
                out = negate(cls_word());
                return true;
            case 's':
                out = cls_space();
                return true;
            case 'S':
                out = negate(cls_space());
                return true;
            case 'l':
                out = cls_lower();
                return true;
            case 'u':
                out = cls_upper();
                return true;
            default:
                return false;
        }
    }

    // single-character escapes; returns byte value or -1
    int char_escape(int c) {
        switch (c) {
            case 'a':
                return 7;
            case 'e':
                return 27;
            case 'f':
                return 12;
            case 'n':
                return 10;
            case 'r':
                return 13;
            case 't':
                return 9;
            case 'x': {
                if (peek() == '{') {
                    ++i;
                    long v = 0;
                    int nd = 0;
                    while (hexval(peek()) >= 0) {
                        v = v * 16 + hexval(p[i++]);
                        ++nd;
                        if (v > 255)
                            throw Unsupported("\\x{...} beyond one byte");
                    }
                    if (peek() != '}' || nd == 0)
                        throw Invalid("bad \\x{}");
                    ++i;
                    return (int)v;
                }
                int v = 0, nd = 0;
                while (nd < 2 && hexval(peek()) >= 0) {
                    v = v * 16 + hexval(p[i++]);
                    ++nd;
                }
                if (nd == 0)
                    throw Invalid("bad \\x");
                return v;
            }
            case 'c': {
                if (!more())
                    throw Invalid("bad \\c");
                int v = p[i++];
                return v & 0x1F;
            }
            case '0': {
                int v = 0, nd = 0;
                while (nd < 3 && peek() >= '0' && peek() <= '7') {
                    v = v * 8 + (p[i++] - '0');
                    ++nd;
                }
                return v & 0xFF;
            }
            default:
                return -1;
        }
    }

    int parse_escape_atom(bool& is_atom) {
        // at char after '\'
        if (!more())
            throw Invalid("trailing backslash");
        int c = p[i++];
        ByteSet cs;
        if (class_escape(c, cs))
            return mk_set(cs);
        if (c == 'h')
            return mk_set(cls_blank());
        if (c == 'H')
            return mk_set(negate(cls_blank()));
        if (c == 'v')
            return mk_set(cls_vspace());
        if (c == 'V')
            return mk_set(negate(cls_vspace()));
        int v = char_escape(c);
        if (v >= 0)
            return mk_byte((unsigned)v);
        if (c >= '1' && c <= '9')
            throw Unsupported("back-reference");
        uint32_t ak = 0;
        switch (c) {
            case 'b':
                ak = A_WORDB;
                break;
            case 'B':
                ak = A_NWORDB;
                break;
            case '<':
                ak = A_WSTART;
                break;
            case '>':
                ak = A_WEND;
                break;
            case 'A':
            case '`':
                ak = A_BOT;
                break;
            case 'z':
            case '\'':
                ak = A_EOT;
                break;
            case 'Q': {
                std::vector<int> items;
                while (more()) {
                    if (p[i] == '\\' && i + 1 < n && p[i + 1] == 'E') {
                        i += 2;
                        break;
                    }
                    items.push_back(mk_byte(p[i++]));
                }
                if (items.empty()) {
                    is_atom = false;
                    return -1;
                }
                if (items.size() == 1)
                    return items[0];
                // a quantifier after \Q..\E applies to the last literal only: keep it simple and reject
                int c2 = peek();
                if (c2 == '*' || c2 == '+' || c2 == '?' || c2 == '{')
                    throw Unsupported("quantifier after \\Q..\\E");
                int id = mk(N_CAT);
                nodes[id].kids = items;
                return id;
            }
            case 'Z':
            case 'G':
            case 'K':
            case 'X':
            case 'C':
            case 'R':
            case 'N':
            case 'p':
            case 'P':
            case 'g':
            case 'k':
            case 'E':
            case 'L':
            case 'U':
                throw Unsupported(std::string("escape \\") + (char)c);
            default:
                break;
        }
        if (ak) {
            is_atom = false;
            int id = mk(N_ASSERT);
            nodes[id].akind = ak;
            return id;
        }
        if ((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z'))
            throw Unsupported(std::string("escape \\") + (char)c);
        return mk_byte((unsigned)c); // escaped punctuation / any other byte: the byte itself
    }

    int parse_set() {
        // at char after '['
        ByteSet s;
        bool neg = false;
        if (peek() == '^') {
            neg = true;
            ++i;
        }
        bool first = true;
        for (;;) {
            if (!more())
                throw Invalid("unterminated character set");
            int c = p[i];
            if (c == ']' && !first) {
                ++i;
                break;
            }
            first = false;
            int lo = -1;
            ByteSet cs;
            bool is_class = false;
            if (c == '[' && i + 1 < n && (p[i + 1] == ':' || p[i + 1] == '.' || p[i + 1] == '=')) {
                int kind = p[i + 1];
                size_t s0 = i + 2, e = s0;
                while (e + 1 < n && !(p[e] == kind && p[e + 1] == ']'))
                    ++e;
                if (e + 1 >= n)
                    throw Invalid("unterminated [: :]");
                std::string name((const char*)p + s0, e - s0);
                i = e + 2;
                if (kind != ':')
                    throw Unsupported("collating element / equivalence class");
                bool nneg = false;
                if (!name.empty() && name[0] == '^') {
                    nneg = true;
                    name = name.substr(1);
                }
                if (name == "alnum")
                    cs = cls_alnum();
                else if (name == "alpha")
                    cs = cls_alpha();
                else if (name == "blank")
                    cs = cls_blank();
                else if (name == "cntrl")
                    cs = cls_cntrl();
                else if (name == "digit" || name == "d")
                    cs = cls_digit();
                else if (name == "graph")
                    cs = cls_graph();
                else if (name == "lower" || name == "l")
                    cs = cls_lower();
                else if (name == "print")
                    cs = cls_print();
                else if (name == "punct")
                    cs = cls_punct();
                else if (name == "space" || name == "s")
                    cs = cls_space();
                else if (name == "upper" || name == "u")
                    cs = cls_upper();
                else if (name == "xdigit")
                    cs = cls_xdigit();
                else if (name == "word" || name == "w")
                    cs = cls_word();
                else
                    throw Invalid("unknown character class name");
                if (nneg)
                    cs.invert();
                is_class = true;
            } else if (c == '\\') {
                ++i;
                if (!more())
                    throw Invalid("trailing backslash in set");
                int e = p[i++];
                if (class_escape(e, cs)) {
                    is_class = true;
                } else {
                    int v = char_escape(e);
                    if (v >= 0) {
                        lo = v;
                    } else if ((e >= 'a' && e <= 'z') || (e >= 'A' && e <= 'Z') || (e >= '1' && e <= '9')) {
                        throw Unsupported(std::string("escape \\") + (char)e + " inside a set");
                    } else {
                        lo = e;
                    }
                }
            } else {
                lo = c;
                ++i;
            }
            if (is_class) {
                if (peek() == '-' && i + 1 < n && p[i + 1] != ']')
                    throw Unsupported("range starting at a class");
                if (icase) {
                    // classes are closed under ASCII case except lower/upper: fold them
                    for (unsigned b = 'a'; b <= 'z'; ++b)
                        if (cs.test(b) || cs.test(b - 32)) {
                            cs.set(b);
                            cs.set(b - 32);
                        }
                }
                s.merge(cs);
                continue;
            }
            int hi = lo;
            if (peek() == '-' && i + 1 < n && p[i + 1] != ']') {
                ++i;
                int c2 = p[i];
                if (c2 == '[' && i + 1 < n && (p[i + 1] == ':' || p[i + 1] == '.' || p[i + 1] == '='))
                    throw Unsupported("range ending at a class");
                if (c2 == '\\') {
                    ++i;
                    if (!more())
                        throw Invalid("trailing backslash in set");
                    int e = p[i++];
                    ByteSet tmp;
                    if (class_escape(e, tmp))
                        throw Unsupported("range ending at a class");
                    int v = char_escape(e);
                    if (v >= 0)
                        hi = v;
                    else if ((e >= 'a' && e <= 'z') || (e >= 'A' && e <= 'Z') || (e >= '1' && e <= '9'))
                        throw Unsupported("escape inside a set");
                    else
                        hi = e;
                } else {
                    hi = c2;
                    ++i;
                }
                if (hi < lo)
                    throw Invalid("invalid range in character set");
            }
            for (int b = lo; b <= hi; ++b) {
                s.set((unsigned)b);
                if (icase) {
                    if (b >= 'a' && b <= 'z')
                        s.set((unsigned)b - 32);
                    if (b >= 'A' && b <= 'Z')
                        s.set((unsigned)b + 32);
                }
            }
        }
        if (neg)
            s.invert();
        int id = mk(N_SET);
        nodes[id].set = s;
        return id;
    }

    int parse_atom(bool& is_atom) {
        int c = p[i];
        switch (c) {
            case '(': {
                int g = parse_group();
                if (g < 0)
                    is_atom = false;
                return g;
            }
            case '[':
                ++i;
                return parse_set();
            case '.': {
                ++i;
                ByteSet s;
                s.invert(); // boost default: '.' matches every char including '\n' and NUL
                int id = mk(N_SET);
                nodes[id].set = s;
                return id;
            }
            case '^': {
                ++i;
                is_atom = false;
                int id = mk(N_ASSERT);
                nodes[id].akind = A_BOL;
                return id;
            }
            case '$': {
                ++i;
                is_atom = false;
                int id = mk(N_ASSERT);
                nodes[id].akind = A_EOL;
                return id;
            }
            case '\\':
                ++i;
                return parse_escape_atom(is_atom);
            case '*':
            case '+':
            case '?':
                throw Invalid("nothing to repeat");
            case '{':
                throw Invalid("unexpected {");
            default:
                ++i;
                return mk_byte((unsigned)c);
        }
    }

    int parse_all() {
        int r = parse_alt();
        if (more()) {
            if (peek() == ')')
                throw Invalid("unmatched )");
            throw Invalid("trailing characters");
        }
        return r;
    }
};

// ------------------------------------------------------------------------------------------ NFA program
enum Op { OP_CHAR, OP_SPLIT, OP_JMP, OP_SAVE, OP_ASSERT, OP_MATCH };
struct Inst {
    Op op;
    int x = -1, y = -1; // CHAR/SAVE/ASSERT/JMP: x = next ; SPLIT: x preferred, y alternative
    int arg = 0;        // CHAR: set id ; SAVE: slot ; ASSERT: kind mask
};

struct Compiler {
    const std::vector<Node>& nodes;
    std::vector<Inst> prog;
    std::vector<ByteSet> sets;
    std::map<ByteSet, int> set_ids;
    size_t max_insts = 6000;

    explicit Compiler(const std::vector<Node>& n) : nodes(n) {}

    int emit(Op op, int arg = 0) {
        if (prog.size() >= max_insts)
            throw Unsupported("pattern too large after expansion");
        Inst in;
        in.op = op;
        in.arg = arg;
        prog.push_back(in);
        return (int)prog.size() - 1;
    }
    int set_id(const ByteSet& s) {
        auto it = set_ids.find(s);
        if (it != set_ids.end())
            return it->second;
        int id = (int)sets.size();
        sets.push_back(s);
        set_ids[s] = id;
        return id;
    }

    bool nullable(int id) const {
        const Node& nd = nodes[id];
        switch (nd.kind) {
            case N_EMPTY:
            case N_ASSERT:
                return true;
            case N_SET:
                return false;
            case N_CAT:
                for (int k : nd.kids)
                    if (!nullable(k))
                        return false;
                return true;
            case N_ALT:
                for (int k : nd.kids)
                    if (nullable(k))
                        return true;
                return false;
            case N_REP:
                return nd.min == 0 || nullable(nd.kids[0]);
            case N_GROUP:
                return nullable(nd.kids[0]);
        }
        return true;
    }

    // A fragment is "open": control falls through to the next emitted instruction; dangling jumps are
    // collected in `outs` and patched by the caller to the instruction that follows the fragment.
    void patch(std::vector<int*>& outs, int target) {
        for (int* o : outs)
            *o = target;
        outs.clear();
    }

    // Emits code for node; on return, every pointer in `holes` must be set to the index of the next
    // instruction emitted after this fragment.  Since `prog` may reallocate we store (inst, field) pairs.
    struct Hole {
        int inst;
        int field; // 0 = x, 1 = y
    };
    void fill(std::vector<Hole>& holes, int target) {
        for (auto h : holes)
            (h.field ? prog[h.inst].y : prog[h.inst].x) = target;
        holes.clear();
    }

    // Returns the list of holes to be pointed at whatever comes next.
    std::vector<Hole> gen(int id) {
        const Node& nd = nodes[id];
        std::vector<Hole> holes;
        switch (nd.kind) {
            case N_EMPTY:
                break;
            case N_SET: {
                if (nd.set.empty()) {
                    // matches nothing: a CHAR over the empty set is a dead end
                }
                int c = emit(OP_CHAR, set_id(nd.set));
                holes.push_back({c, 0});
                break;
            }
            case N_ASSERT: {
                int a = emit(OP_ASSERT, (int)nd.akind);
                holes.push_back({a, 0});
                break;
            }
            case N_GROUP: {
                if (nd.cap >= 0) {
                    int s0 = emit(OP_SAVE, 2 * (nd.cap - 1));
                    std::vector<Hole> h0 = {{s0, 0}};
                    fill(h0, (int)prog.size());
                    auto h = gen(nd.kids[0]);
                    int s1 = emit(OP_SAVE, 2 * (nd.cap - 1) + 1);
                    fill(h, s1);
                    holes.push_back({s1, 0});
                } else {
                    holes = gen(nd.kids[0]);
                }
                break;
            }
            case N_CAT: {
                std::vector<Hole> pending;
                for (int k : nd.kids) {
                    fill(pending, (int)prog.size());
                    pending = gen(k);
                }
                holes = pending;
                break;
            }
            case N_ALT: {
                // split chain preferring earlier alternatives
                size_t na = nd.kids.size();
                for (size_t a = 0; a < na; ++a) {
                    if (a + 1 < na) {
                        int sp = emit(OP_SPLIT);
                        prog[sp].x = (int)prog.size();
                        auto h = gen(nd.kids[a]);
                        // the alternative may be empty (no instruction emitted): then x already points at
                        // the next instruction, which is wrong -- route it through an explicit JMP hole
                        int j = emit(OP_JMP);
                        fill(h, j);
                        holes.push_back({j, 0});
                        prog[sp].y = (int)prog.size();
                    } else {
                        auto h = gen(nd.kids[a]);
                        int j = emit(OP_JMP);
                        fill(h, j);
                        holes.push_back({j, 0});
                    }
                }
                break;
            }
            case N_REP: {
                int child = nd.kids[0];
                if ((nd.max < 0 || nd.max > 1) && nullable(child))
                    throw Unsupported("repeat of a sub-expression that can match the empty string");
                std::vector<Hole> pending;
                for (int r = 0; r < nd.min; ++r) {
                    fill(pending, (int)prog.size());
                    pending = gen(child);
                }
                if (nd.max < 0) {
                    // star:  L: SPLIT body, exit ; body ; JMP L
                    int sp = emit(OP_SPLIT);
                    fill(pending, sp);
                    int body = (int)prog.size();
                    auto h = gen(child);
                    int j = emit(OP_JMP);
                    fill(h, j);
                    prog[j].x = sp;
                    if (nd.greedy) {
                        prog[sp].x = body;
                        holes.push_back({sp, 1});
                    } else {
                        prog[sp].y = body;
                        holes.push_back({sp, 0});
                    }
                } else {
                    // (max - min) nested optionals, all skipping to the common end
                    for (int r = nd.min; r < nd.max; ++r) {
                        int sp = emit(OP_SPLIT);
                        fill(pending, sp);
                        int body = (int)prog.size();
                        pending = gen(child);
                        if (pending.empty() && body == (int)prog.size()) {
                            // empty body: nothing emitted
                        }
                        if (nd.greedy) {
                            prog[sp].x = body;
                            holes.push_back({sp, 1});
                        } else {
                            prog[sp].y = body;
                            holes.push_back({sp, 0});
                        }
                    }
                    for (auto h : pending)
                        holes.push_back(h);
                }
                break;
            }
        }
        return holes;
    }
};

// ------------------------------------------------------------------------------------------ context kinds
enum Kind { K_EDGE = 0, K_LF = 1, K_CR = 2, K_FF = 3, K_WORD = 4, K_OTHER = 5, K_COUNT = 6 };

int byte_kind(unsigned b) {
    if (b == '\n')
        return K_LF;
    if (b == '\r')
        return K_CR;
    if (b == '\f')
        return K_FF;
    if ((b >= '0' && b <= '9') || (b >= 'a' && b <= 'z') || (b >= 'A' && b <= 'Z') || b == '_')
        return K_WORD;
    return K_OTHER;
}

// boost perl_matcher::match_start_line / match_end_line / match_word_boundary semantics on (prev kind, next kind);
// K_EDGE means start of input (prev) or end of input (next).
bool asserts_hold(uint32_t mask, int pk, int nk) {
    auto sep = [](int k) { return k == K_LF || k == K_CR || k == K_FF; };
    if (mask & A_BOL) {
        if (!(pk == K_EDGE || (sep(pk) && !(pk == K_CR && nk == K_LF))))
            return false;
    }
    if (mask & A_EOL) {
        if (!(nk == K_EDGE || (sep(nk) && !(pk == K_CR && nk == K_LF))))
            return false;
    }
    if ((mask & A_BOT) && pk != K_EDGE)
        return false;
    if ((mask & A_EOT) && nk != K_EDGE)
        return false;
    if (mask & A_WORDB) {
        if ((pk == K_WORD) == (nk == K_WORD))
            return false;
    }
    // perl_matcher::match_word_start / match_word_end (boost 1.68 perl_matcher_common.hpp): \< needs a word byte next
    // (never at the end of the buffer) and no word byte before it; \> needs a word byte before it (never at the start)
    // and no word byte next
    if ((mask & A_WSTART) && !(nk == K_WORD && pk != K_WORD))
        return false;
    if ((mask & A_WEND) && !(pk == K_WORD && nk != K_WORD))
        return false;
    if (mask & A_NWORDB) {
        // perl_matcher::match_within_word (boost 1.68 perl_matcher_common.hpp): false at either edge of the buffer
        // (position == last, or position == backstop without match_prev_avail) -- unlike Perl / PCRE, which let \B
        // hold at an edge next to a non-word character -- else both neighbours are word characters or both are not
        if (pk == K_EDGE || nk == K_EDGE || (pk == K_WORD) != (nk == K_WORD))
            return false;
    }
    return true;
}

struct Cand {
    int target; // walker index (>=1) of a CHAR inst, or -1 for MATCH
    uint64_t saves;
    uint32_t asserts;
};

template <class T>
void put(std::vector<uint8_t>& blob, uint32_t& off_field, const std::vector<T>& v) {
    while (blob.size() % 16)
        blob.push_back(0);
    off_field = (uint32_t)blob.size();
    const uint8_t* p = (const uint8_t*)v.data();
    blob.insert(blob.end(), p, p + v.size() * sizeof(T));
}

} // namespace

CompileResult compile_regex(const char* pattern, size_t len, size_t max_table_bytes) {
    CompileResult res;
    try {
        Parser ps(pattern, len);
        int root = ps.parse_all();
        res.valid = true;
        res.ngroups = (uint32_t)ps.ncap;
        if (ps.ncap > (int)LC_MAX_GROUPS)
            throw Unsupported("more than 32 capture groups");

        Compiler cc(ps.nodes);
        auto holes = cc.gen(root);
        int m = cc.emit(OP_MATCH);
        cc.fill(holes, m);
        const std::vector<Inst>& prog = cc.prog;
        res.n_insts = (uint32_t)prog.size();

        bool has_ctx = false; // any assertion at all: byte classes are refined by context kind
        for (auto& in : prog)
            if (in.op == OP_ASSERT)
                has_ctx = true;
        auto kind_of = [&](unsigned b) { return has_ctx ? byte_kind(b) : 0; };

        // ---- walker states: 0 = START, 1.. = CHAR instructions
        std::vector<int> walker_of(prog.size(), -1), inst_of_walker = {-1};
        for (size_t k = 0; k < prog.size(); ++k)
            if (prog[k].op == OP_CHAR) {
                walker_of[k] = (int)inst_of_walker.size();
                inst_of_walker.push_back((int)k);
            }
        const int nw = (int)inst_of_walker.size();
        if (nw > 4000)
            throw Unsupported("too many NFA states");
        res.n_walkers = (uint32_t)nw;

        // ---- priority-ordered candidate lists
        std::vector<std::vector<Cand>> cand(nw);
        {
            std::vector<std::vector<uint32_t>> seen;
            std::vector<Cand>* out = nullptr;
            size_t budget = 0;
            struct Rec {
                const std::vector<Inst>& prog;
                const std::vector<int>& walker_of;
                std::vector<std::vector<uint32_t>>& seen;
                std::vector<Cand>*& out;
                size_t& budget;
                void go(int pc, uint64_t saves, uint32_t am) {
                    if (++budget > 2000000)
                        throw Unsupported("epsilon closure too large");
                    for (uint32_t mk : seen[pc])
                        if ((mk & am) == mk)
                            return; // an earlier (higher priority) arrival dominates
                    seen[pc].push_back(am);
                    const Inst& in = prog[pc];
                    switch (in.op) {
                        case OP_CHAR:
                            out->push_back({walker_of[pc], saves, am});
                            break;
                        case OP_MATCH:
                            out->push_back({-1, saves, am});
                            break;
                        case OP_JMP:
                            go(in.x, saves, am);
                            break;
                        case OP_SPLIT:
                            go(in.x, saves, am);
                            go(in.y, saves, am);
                            break;
                        case OP_SAVE:
                            go(in.x, saves | (1ull << in.arg), am);
                            break;
                        case OP_ASSERT:
                            go(in.x, saves, am | (uint32_t)in.arg);
                            break;
                    }
                }
            } rec{prog, walker_of, seen, out, budget};
            for (int w = 0; w < nw; ++w) {
                seen.assign(prog.size(), {});
                out = &cand[w];
                budget = 0;
                int entry = (w == 0) ? 0 : prog[inst_of_walker[w]].x;
                rec.go(entry, 0, 0);
            }
        }

        // ---- static resolution of assertions whose context is fixed.
        // START always stands at offset 0 (prev == EDGE): ^ and \A hold.  Every automaton strips those.
        for (auto& cd : cand[0])
            cd.asserts &= ~(uint32_t)(A_BOL | A_BOT);
        // The PREFIX dfa keeps everything else; the full-match automata additionally know that MATCH is only
        // ever taken at end of input (next == EDGE): $ and \z hold there.
        std::vector<std::vector<Cand>> cand_prefix = cand;
        bool ctx_prefix = false, ctx_full = false;
        for (auto& lst : cand)
            for (auto& cd : lst) {
                if (cd.asserts)
                    ctx_prefix = true;
                if (cd.target < 0)
                    cd.asserts &= ~(uint32_t)(A_EOL | A_EOT);
                if (cd.asserts)
                    ctx_full = true;
            }
        const int npc = ctx_full ? K_COUNT : 1;

        // ---- byte classes
        uint8_t byte_class[256];
        int nclasses = 0;
        {
            std::map<std::vector<uint8_t>, int> sig_to_class;
            for (unsigned b = 0; b < 256; ++b) {
                std::vector<uint8_t> sig;
                sig.reserve(cc.sets.size() + 1);
                for (auto& s : cc.sets)
                    sig.push_back(s.test(b));
                for (auto& la : ps.las) // a look-ahead set is a union of classes
                    sig.push_back(la.set.test(b));
                sig.push_back((uint8_t)kind_of(b));
                auto it = sig_to_class.find(sig);
                if (it == sig_to_class.end()) {
                    it = sig_to_class.emplace(sig, nclasses++).first;
                }
                byte_class[b] = (uint8_t)it->second;
            }
        }
        std::vector<unsigned> class_rep(nclasses); // a representative byte
        for (int b = 255; b >= 0; --b)
            class_rep[byte_class[b]] = (unsigned)b;
        std::vector<uint8_t> class_kind(nclasses);
        for (int c = 0; c < nclasses; ++c)
            class_kind[c] = (uint8_t)kind_of(class_rep[c]);
        auto walker_has = [&](int w, int c) { return cc.sets[prog[inst_of_walker[w]].arg].test(class_rep[c]); };
        // Single-byte look-aheads look at the NEXT byte itself, not only at its kind: where the automata carry the
        // "next" context in their states (the reverse DFA) it is the byte CLASS + 1 (0 = end of input) instead of the
        // kind when the pattern has such assertions; forward automata know the class of the byte they are consuming.
        const bool has_la = !ps.las.empty();
        auto ctx_kind = [&](int ctx) { return has_la ? (ctx == 0 ? (int)K_EDGE : (int)class_kind[ctx - 1]) : ctx; };
        auto ctx_class = [&](int ctx) { return has_la ? ctx - 1 : -2; }; // -1 = end of input, -2 = not tracked
        auto ctx_of_class = [&](int c) { return has_la ? c + 1 : (int)class_kind[c]; };
        // all assertions of `mask` with previous kind pk, next kind nk and next class ncls (-1 = end of input)
        auto holds = [&](uint32_t mask, int pk, int nk, int ncls) {
            if (!asserts_hold(mask, pk, nk))
                return false;
            for (size_t q = 0; q < ps.las.size(); ++q)
                if (mask & (A_LA0 << q)) {
                    if (ncls == -2)
                        throw Unsupported("look-ahead in this automaton");
                    const bool member = ncls >= 0 && ps.las[q].set.test(class_rep[ncls]);
                    if (member == ps.las[q].neg)
                        return false;
                }
            return true;
        };
        // kinds the byte consumed by walker w can have (prev context when standing in w)
        std::vector<uint32_t> walker_pcs(nw, 0);
        walker_pcs[0] = 1u << 0; // START: K_EDGE (or the single collapsed kind)
        for (int w = 1; w < nw; ++w)
            for (int c = 0; c < nclasses; ++c)
                if (walker_has(w, c))
                    walker_pcs[w] |= 1u << class_kind[c];

        // ---- actions
        std::vector<uint64_t> actions = {0};
        std::map<uint64_t, uint32_t> action_id = {{0ull, 0u}};
        auto act = [&](uint64_t mask) {
            auto it = action_id.find(mask);
            if (it != action_id.end())
                return it->second;
            uint32_t id = (uint32_t)actions.size();
            if (id >= 0xFFFF)
                throw Unsupported("too many distinct capture actions");
            actions.push_back(mask);
            action_id[mask] = id;
            return id;
        };
        auto entry_of = [&](const Cand& cd) {
            uint32_t nxt = cd.target < 0 ? 0xFFFFu : (uint32_t)cd.target;
            return nxt | (act(cd.saves) << 16);
        };

        // ---- PREFIX dfa (forward subset construction; boolean, order-insensitive)
        std::vector<uint16_t> pre_next;
        std::vector<uint8_t> pre_acc;
        uint32_t pre_start = 1;
        {
            typedef std::pair<std::vector<int>, int> Key; // (sorted walker set, prev kind)
            std::map<Key, uint32_t> ids;
            std::vector<Key> states;
            states.push_back(Key()); // 0 = dead
            auto intern = [&](Key k) -> uint32_t {
                if (k.first.empty())
                    return 0;
                auto it = ids.find(k);
                if (it != ids.end())
                    return it->second;
                if (states.size() >= 8000)
                    throw Unsupported("prefix DFA too large");
                uint32_t id = (uint32_t)states.size();
                ids[k] = id;
                states.push_back(k);
                return id;
            };
            pre_start = intern(Key({0}, 0));
            for (size_t s = 0; s < states.size(); ++s) {
                pre_next.resize((s + 1) * nclasses, 0);
                pre_acc.resize(s + 1, 0);
                if (s == 0)
                    continue;
                Key cur = states[s]; // copy: `states` grows
                int pk = cur.second;
                for (int w : cur.first)
                    for (auto& cd : cand_prefix[w])
                        if (cd.target < 0 && holds(cd.asserts, pk, K_EDGE, -1))
                            pre_acc[s] = 1;
                for (int c = 0; c < nclasses; ++c) {
                    int nk = class_kind[c];
                    bool accept_now = false;
                    std::set<int> nxt;
                    for (int w : cur.first)
                        for (auto& cd : cand_prefix[w]) {
                            if (cd.asserts && !holds(cd.asserts, pk, nk, c))
                                continue;
                            if (cd.target < 0)
                                accept_now = true;
                            else if (walker_has(cd.target, c))
                                nxt.insert(cd.target);
                        }
                    uint32_t v;
                    if (accept_now)
                        v = LC_PREFIX_ACCEPT;
                    else
                        v = intern(Key(std::vector<int>(nxt.begin(), nxt.end()), ctx_prefix ? nk : 0));
                    pre_next[s * nclasses + c] = (uint16_t)v;
                }
            }
            res.n_prefix = (uint32_t)states.size();
        }
        // NB: a zero assertion mask always holds, so context kinds are irrelevant wherever masks were stripped.

        // ---- reverse DFA over viable-target sets
        // state = (sorted set of targets {walker idx, or 0 for MATCH}, next kind)
        typedef std::pair<std::vector<int>, int> RKey;
        std::vector<RKey> rstates;
        std::vector<uint16_t> rev_next;
        std::vector<std::vector<uint8_t>> rev_incoming; // classes on which each state is entered
        uint32_t rev_start = 1;
        {
            std::map<RKey, uint32_t> ids;
            rstates.push_back(RKey()); // 0 dead
            auto intern = [&](RKey k) -> uint32_t {
                if (k.first.empty())
                    return 0;
                auto it = ids.find(k);
                if (it != ids.end())
                    return it->second;
                if (rstates.size() >= 8000)
                    throw Unsupported("reverse DFA too large");
                uint32_t id = (uint32_t)rstates.size();
                ids[k] = id;
                rstates.push_back(k);
                return id;
            };
            rev_start = intern(RKey({0}, 0)); // {MATCH}, next = EDGE
            for (size_t s = 0; s < rstates.size(); ++s) {
                rev_next.resize((s + 1) * nclasses, 0);
                rev_incoming.resize(rstates.size());
                if (s == 0)
                    continue;
                RKey cur = rstates[s];
                std::vector<char> inR(nw, 0);
                bool match_in = false;
                for (int t : cur.first) {
                    if (t == 0)
                        match_in = true;
                    else
                        inR[t] = 1;
                }
                const int nk = ctx_kind(cur.second), nkc = ctx_class(cur.second);
                for (int c = 0; c < nclasses; ++c) {
                    int pk = class_kind[c];
                    std::vector<int> nxt;
                    for (int q = 1; q < nw; ++q) {
                        if (!walker_has(q, c))
                            continue;
                        bool viable = false;
                        for (auto& cd : cand[q]) {
                            bool in = cd.target < 0 ? match_in : (bool)inR[cd.target];
                            if (in && holds(cd.asserts, pk, nk, nkc)) {
                                viable = true;
                                break;
                            }
                        }
                        if (viable)
                            nxt.push_back(q);
                    }
                    uint32_t v = intern(RKey(nxt, ctx_full ? ctx_of_class(c) : 0));
                    rev_next[s * nclasses + c] = (uint16_t)v;
                    rev_incoming.resize(rstates.size());
                    if (v)
                        rev_incoming[v].push_back((uint8_t)c);
                }
            }
            res.n_rev = (uint32_t)rstates.size();
        }
        const int nD = (int)rstates.size();

        // first viable candidate of walker w under prev kind pk in reverse state D (index into cand[w] or -1)
        auto first_viable = [&](int w, int pk, int D) -> int {
            const RKey& k = rstates[D];
            for (size_t ci = 0; ci < cand[w].size(); ++ci) {
                const Cand& cd = cand[w][ci];
                int t = cd.target < 0 ? 0 : cd.target;
                if (std::binary_search(k.first.begin(), k.first.end(), t) &&
                    holds(cd.asserts, pk, ctx_kind(k.second), ctx_class(k.second)))
                    return (int)ci;
            }
            return -1;
        };
        // first class-compatible candidate (forward-only choice)
        auto first_fwd = [&](int w, int pk, int c /* class or -1 for EOF */) -> int {
            int nk = c < 0 ? K_EDGE : class_kind[c];
            for (size_t ci = 0; ci < cand[w].size(); ++ci) {
                const Cand& cd = cand[w][ci];
                if (cd.asserts && !holds(cd.asserts, pk, nk, c < 0 ? -1 : c))
                    continue;
                if (c < 0) {
                    if (cd.target < 0)
                        return (int)ci;
                } else if (cd.target >= 0 && walker_has(cd.target, c)) {
                    return (int)ci;
                }
            }
            return -1;
        };

        // ---- is the forward-only automaton exact?
        bool fwd1_safe = true;
        for (int D = 1; D < nD && fwd1_safe; ++D) {
            for (int w = 0; w < nw && fwd1_safe; ++w) {
                for (int pk = 0; pk < npc && fwd1_safe; ++pk) {
                    if (npc > 1 && !(walker_pcs[w] >> pk & 1))
                        continue;
                    int v = first_viable(w, pk, D);
                    if (v < 0)
                        continue;
                    if ((uint32_t)D == rev_start) {
                        if (first_fwd(w, pk, -1) != v)
                            fwd1_safe = false;
                    }
                    for (uint8_t c : rev_incoming[D])
                        if (first_fwd(w, pk, c) != v) {
                            fwd1_safe = false;
                            break;
                        }
                }
            }
        }

        // ---- forward tables
        std::vector<uint32_t> fwd, fwd_eof;
        uint32_t fwd_cols;
        uint32_t mode;
        if (fwd1_safe) {
            mode = LC_MODE_FWD1;
            fwd_cols = (uint32_t)nclasses;
            fwd.assign((size_t)nw * npc * fwd_cols, LC_NONE_ENTRY);
            fwd_eof.assign((size_t)nw * npc, LC_NONE_ENTRY);
            for (int w = 0; w < nw; ++w)
                for (int pk = 0; pk < npc; ++pk) {
                    for (int c = 0; c < nclasses; ++c) {
                        int ci = first_fwd(w, pk, c);
                        if (ci >= 0)
                            fwd[((size_t)w * npc + pk) * fwd_cols + c] = entry_of(cand[w][ci]);
                    }
                    int ci = first_fwd(w, pk, -1);
                    if (ci >= 0)
                        fwd_eof[(size_t)w * npc + pk] = entry_of(cand[w][ci]);
                }
        } else {
            mode = LC_MODE_TWOPASS;
            fwd_cols = (uint32_t)nD;
            if ((size_t)nw * npc * fwd_cols * 4 > max_table_bytes)
                throw Unsupported("two-pass forward table too large");
            fwd.assign((size_t)nw * npc * fwd_cols, LC_NONE_ENTRY);
            fwd_eof.assign((size_t)nw * npc, LC_NONE_ENTRY);
            for (int w = 0; w < nw; ++w)
                for (int pk = 0; pk < npc; ++pk)
                    for (int D = 1; D < nD; ++D) {
                        int ci = first_viable(w, pk, D);
                        if (ci >= 0)
                            fwd[((size_t)w * npc + pk) * fwd_cols + D] = entry_of(cand[w][ci]);
                    }
        }

        // ---- pack the blob
        LcRegexHeader h;
        memset(&h, 0, sizeof h);
        h.magic = LC_REGEX_MAGIC;
        h.ngroups = res.ngroups;
        h.nclasses = (uint32_t)nclasses;
        h.mode = mode;
        h.npc = (uint32_t)npc;
        h.nw = (uint32_t)nw;
        h.nact = (uint32_t)actions.size();
        h.pre_nstates = res.n_prefix;
        h.pre_start = pre_start;
        h.rev_nstates = (uint32_t)nD;
        h.rev_start = rev_start;
        h.fwd_cols = fwd_cols;
        std::vector<uint8_t> blob(sizeof h, 0);
        std::vector<uint8_t> bc(byte_class, byte_class + 256);
        put(blob, h.off_byte_class, bc);
        put(blob, h.off_class_pc, class_kind);
        put(blob, h.off_actions, actions);
        put(blob, h.off_pre_next, pre_next);
        put(blob, h.off_pre_acc, pre_acc);
        put(blob, h.off_fwd, fwd);
        put(blob, h.off_fwd_eof, fwd_eof);
        if (mode == LC_MODE_TWOPASS) {
            put(blob, h.off_rev_next, rev_next);
            h.rev_label_bytes = nD <= 256 ? 1 : 2;
            if (nD <= 256) {
                std::vector<uint8_t> rb((size_t)nD * 256);
                for (int d = 0; d < nD; ++d)
                    for (int b = 0; b < 256; ++b)
                        rb[(size_t)d * 256 + b] = (uint8_t)rev_next[(size_t)d * nclasses + byte_class[b]];
                put(blob, h.off_rev_byte, rb);
            } else {
                std::vector<uint16_t> rb((size_t)nD * 256);
                for (int d = 0; d < nD; ++d)
                    for (int b = 0; b < 256; ++b)
                        rb[(size_t)d * 256 + b] = rev_next[(size_t)d * nclasses + byte_class[b]];
                put(blob, h.off_rev_byte, rb);
            }
        } else if (npc == 1) {
            std::vector<uint32_t> fb((size_t)nw * 256);
            for (int w = 0; w < nw; ++w)
                for (int b = 0; b < 256; ++b)
                    fb[(size_t)w * 256 + b] = fwd[(size_t)w * fwd_cols + byte_class[b]];
            put(blob, h.off_fwd_byte, fb);
        }
        while (blob.size() % 16)
            blob.push_back(0);
        h.total_bytes = (uint32_t)blob.size();
        memcpy(blob.data(), &h, sizeof h);
        if (blob.size() > max_table_bytes)
            throw Unsupported("automaton tables too large");
        res.blob.swap(blob);
        res.supported = true;

        // ---- kernel-ready "fast" layout (see lc_tables.h)
        if (mode == LC_MODE_TWOPASS && npc == 1 && (uint32_t)nD <= LC_FAST_MAX_REV &&
            (uint32_t)nw <= LC_FAST_MAX_WALKERS && res.ngroups <= LC_FAST_MAX_GROUPS && actions.size() < 256) {
            LcFastHeader fh;
            memset(&fh, 0, sizeof fh);
            fh.magic = LC_FAST_MAGIC;
            fh.ngroups = res.ngroups;
            fh.rev_start4 = rev_start * 4;
            fh.nrev = (uint32_t)nD;
            fh.nw = (uint32_t)nw;
            fh.nact = (uint32_t)actions.size();
            std::vector<uint8_t> rv((size_t)nD * LC_FAST_REV_PITCH, 0);
            for (int d = 0; d < nD; ++d)
                for (int b = 0; b < 256; ++b)
                    rv[(size_t)d * LC_FAST_REV_PITCH + b] =
                        (uint8_t)(4 * rev_next[(size_t)d * nclasses + byte_class[b]]);
            std::vector<uint32_t> fw((size_t)nw * 64, LC_NONE_ENTRY);
            std::vector<uint8_t> cx((size_t)nw * 64, 0);
            for (int w = 0; w < nw; ++w)
                for (int D = 0; D < nD; ++D) {
                    uint32_t e = fwd[(size_t)w * fwd_cols + D];
                    if (e == LC_NONE_ENTRY)
                        continue;
                    uint32_t nxt = LC_ENTRY_NEXT(e);
                    uint32_t a = LC_ENTRY_ACT(e);
                    uint64_t mk = actions[a];
                    uint32_t slot_byte = 0, multi_flag = 0;
                    if (mk) {
                        if ((mk & (mk - 1)) == 0) {
                            int bit = 0;
                            while (!(mk >> bit & 1))
                                ++bit;
                            slot_byte = 4u * (uint32_t)bit + 4u;
                        } else {
                            multi_flag = 0x80000000u; // several slots: out-of-line path, action id in cx
                            cx[(size_t)w * 64 + D] = (uint8_t)a;
                            fh.reserved[0] = 1;       // has_multi
                        }
                    }
                    fw[(size_t)w * 64 + D] = slot_byte | ((nxt == 0xFFFFu ? 0u : nxt) << 8) | multi_flag;
                }
            std::vector<uint8_t> fb(sizeof fh, 0);
            put(fb, fh.off_rev, rv);
            while (fb.size() % 256) // forward rows are addressed by OR-ing the label into the row base
                fb.push_back(0);
            put(fb, fh.off_fwd, fw);
            put(fb, fh.off_cx, cx);
            put(fb, fh.off_masks, actions);
            while (fb.size() % 16)
                fb.push_back(0);
            fh.total_bytes = (uint32_t)fb.size();
            memcpy(fb.data(), &fh, sizeof fh);
            res.fast_blob.swap(fb);
        }
        // ---- stride-2 layout (see lc_tables.h: LcFast2Header)
        if (mode == LC_MODE_TWOPASS && npc == 1 && (uint32_t)nD <= 255 && (uint32_t)nw <= 255 &&
            res.ngroups <= LC_FAST_MAX_GROUPS && actions.size() < 65535 &&
            (uint64_t)nD * nclasses * nclasses * 4 < 65536) {
            const uint32_t ncl = (uint32_t)nclasses;
            auto delta = [&](uint32_t D, uint32_t c) -> uint32_t { return rev_next[(size_t)D * ncl + c]; };
            // pair ids over (label(q), label(q+1)) combinations the reverse DFA can produce
            std::vector<uint8_t> pid((size_t)nD * nD, 0);
            std::vector<uint8_t> pair_l(2, 0); // id 0 = impossible
            bool fits = true;
            for (int Lb = 1; Lb < nD && fits; ++Lb)
                for (uint32_t c = 0; c < ncl && fits; ++c) {
                    uint32_t La = delta((uint32_t)Lb, c);
                    if (!La || pid[(size_t)La * nD + Lb])
                        continue;
                    if (pair_l.size() / 2 >= 256) {
                        fits = false;
                        break;
                    }
                    pid[(size_t)La * nD + Lb] = (uint8_t)(pair_l.size() / 2);
                    pair_l.push_back((uint8_t)La);
                    pair_l.push_back((uint8_t)Lb);
                }
            if (fits) {
                const uint32_t npairs = (uint32_t)pair_l.size() / 2;
                LcFast2Header fh;
                memset(&fh, 0, sizeof fh);
                fh.magic = LC_FAST2_MAGIC;
                fh.ngroups = res.ngroups;
                fh.rev_start = rev_start;
                fh.nrev = (uint32_t)nD;
                fh.ncls = ncl;
                fh.nw = (uint32_t)nw;
                fh.npairs = npairs;
                fh.nact = (uint32_t)actions.size();
                fh.row_bytes = ncl * ncl * 4;
                std::vector<uint8_t> cls(byte_class, byte_class + 256);
                const uint32_t pshift = npairs <= 63 ? 2u : 0u;
                const uint32_t f2row = pshift ? 64u : 256u;
                fh.pair_shift = pshift;
                fh.f2_row = f2row;
                for (auto& x : pid)
                    x = (uint8_t)(x << pshift);
                std::vector<uint32_t> t2((size_t)nD * ncl * ncl, 0);
                for (int D = 1; D < nD; ++D)
                    for (uint32_t c1 = 0; c1 < ncl; ++c1) {
                        uint32_t Lb = delta((uint32_t)D, c1);
                        if (!Lb)
                            continue;
                        for (uint32_t c0 = 0; c0 < ncl; ++c0) {
                            uint32_t La = delta(Lb, c0);
                            if (!La)
                                continue;
                            t2[((size_t)D * ncl + c1) * ncl + c0] =
                                (La * fh.row_bytes) | ((uint32_t)pid[(size_t)La * nD + Lb] << 16); // pid is pre-shifted
                        }
                    }
                std::vector<uint8_t> rev1((size_t)nD * ncl, 0);
                for (int D = 0; D < nD; ++D)
                    for (uint32_t c = 0; c < ncl; ++c)
                        rev1[(size_t)D * ncl + c] = (uint8_t)delta((uint32_t)D, c);
                // forward pair tables
                const uint32_t kMulti = 0xFFFFu;
                auto slot_code = [&](uint32_t act_id) -> uint32_t {
                    uint64_t mk = actions[act_id];
                    if (!mk)
                        return 0;
                    if (mk & (mk - 1))
                        return kMulti;
                    int bit = 0;
                    while (!(mk >> bit & 1))
                        ++bit;
                    return 2u * (uint32_t)bit + 2u;
                };
                std::vector<uint32_t> f2((size_t)nw * f2row, 0);
                for (int w = 0; w < nw; ++w)
                    for (uint32_t P = 1; P < npairs; ++P) {
                        uint32_t La = pair_l[2 * P], Lb = pair_l[2 * P + 1];
                        uint32_t e1 = fwd[(size_t)w * fwd_cols + La];
                        if (e1 == LC_NONE_ENTRY || LC_ENTRY_NEXT(e1) == 0xFFFFu)
                            continue; // not viable / MATCH cannot be followed by another step
                        uint32_t w1 = LC_ENTRY_NEXT(e1);
                        uint32_t e2 = fwd[(size_t)w1 * fwd_cols + Lb];
                        if (e2 == LC_NONE_ENTRY)
                            continue;
                        uint32_t w2 = LC_ENTRY_NEXT(e2) == 0xFFFFu ? 0u : LC_ENTRY_NEXT(e2);
                        uint32_t sa = slot_code(LC_ENTRY_ACT(e1)), sb = slot_code(LC_ENTRY_ACT(e2));
                        if (sa == kMulti || sb == kMulti) {
                            fh.has_multi = 1;
                            f2[(size_t)w * f2row + P] = w2 | LC_FAST2_ACT_MULTI;
                        } else {
                            f2[(size_t)w * f2row + P] = w2 | (sa << 8) | (sb << 16);
                        }
                    }
                std::vector<uint32_t> fwd1((size_t)nw * nD, LC_NONE_ENTRY);
                for (int w = 0; w < nw; ++w)
                    for (int D = 0; D < nD; ++D)
                        fwd1[(size_t)w * nD + D] = fwd[(size_t)w * fwd_cols + D];
                std::vector<uint8_t> fb(sizeof fh, 0);
                put(fb, fh.off_cls, cls);
                put(fb, fh.off_t2, t2);
                put(fb, fh.off_pid, pid);
                put(fb, fh.off_pair_l, pair_l);
                put(fb, fh.off_rev1, rev1);
                put(fb, fh.off_f2, f2);
                put(fb, fh.off_fwd1, fwd1);
                put(fb, fh.off_masks, actions);
                while (fb.size() % 16)
                    fb.push_back(0);
                fh.total_bytes = (uint32_t)fb.size();
                memcpy(fb.data(), &fh, sizeof fh);
                res.fast2_blob.swap(fb);
            }
        }

        // ---- single-pass tagged DFA (see lc_tables.h: LcTdfaHeader).  Determinises the priority-ordered thread
        // list of the backtracking search: thread order = priority, the first thread to reach a walker owns it,
        // and the first thread (in order) that can take MATCH at end of input is the boost/Perl answer.
        [&]() {
            const uint32_t ncl = (uint32_t)nclasses;
            const uint32_t T = 2 * res.ngroups;
            // NB: the row pitch is deliberately NOT rounded to a power of two (measured: with 512-byte rows the same
            // class pair of different states always shares a bank and the look-ups conflict; slower on C2)
            // Instead the pitch is an ODD number of words, so that the same class pair of different states falls
            // into different banks.
            const uint64_t row_bytes = (uint64_t)((ncl * ncl) | 1u) * 4;
            if (T > LC_TDFA_MAX_REGS || row_bytes > 16384)
                return;
            // next_state * row_bytes must fit 16 bits even after the kernel rebases the rows to absolute
            // shared-memory addresses: the pair table starts on a row_bytes boundary within the first
            // LC_TDFA_REBASE_ROOM + row_bytes bytes of the window, and one more row is the slow-path sink
            if ((65535 - LC_TDFA_REBASE_ROOM) / row_bytes < 4)
                return;
            const size_t max_states = (size_t)((65535 - LC_TDFA_REBASE_ROOM) / row_bytes) - 2;
            struct TThread {
                int w;
                std::vector<int16_t> reg; // tag -> register, -1 = unset
            };
            struct TState {
                int pk;
                std::vector<TThread> th;
            };
            std::vector<TState> states(1); // 0 = dead
            std::map<std::vector<int16_t>, uint32_t> ids;
            auto key_of = [&](const TState& st) {
                std::vector<int16_t> k;
                k.reserve(1 + st.th.size() * (T + 1));
                k.push_back((int16_t)st.pk);
                for (auto& th : st.th) {
                    k.push_back((int16_t)th.w);
                    k.insert(k.end(), th.reg.begin(), th.reg.end());
                }
                return k;
            };
            bool ok = true;
            auto intern = [&](TState&& st) -> uint32_t {
                if (st.th.empty())
                    return 0;
                auto k = key_of(st);
                auto it = ids.find(k);
                if (it != ids.end())
                    return it->second;
                if (states.size() >= max_states || states.size() >= 4096) {
                    ok = false;
                    return 0;
                }
                uint32_t id = (uint32_t)states.size();
                ids.emplace(std::move(k), id);
                states.push_back(std::move(st));
                return id;
            };
            std::vector<uint16_t> ops = {0}; // list 0 = empty
            std::map<std::vector<uint16_t>, uint32_t> op_ids;
            op_ids[std::vector<uint16_t>()] = 0;
            auto op_list = [&](const std::vector<uint16_t>& lst) -> uint32_t {
                auto it = op_ids.find(lst);
                if (it != op_ids.end())
                    return it->second;
                if (ops.size() + lst.size() + 1 > 65535) {
                    ok = false;
                    return 0;
                }
                uint32_t id = (uint32_t)ops.size();
                ops.push_back((uint16_t)lst.size());
                ops.insert(ops.end(), lst.begin(), lst.end());
                op_ids[lst] = id;
                return id;
            };
            {
                TState st0;
                st0.pk = 0; // K_EDGE (or the single collapsed kind)
                st0.th.push_back({0, std::vector<int16_t>(T, (int16_t)-1)});
                intern(std::move(st0));
            }
            std::vector<uint32_t> t1;                     // [state][class] next | oplist << 16
            std::vector<std::vector<uint8_t>> sets;       // [state][class] registers set by the step
            std::vector<uint32_t> eof;
            uint32_t nregs = T, max_threads = 1;
            for (size_t s = 0; s < states.size() && ok; ++s) {
                t1.resize((s + 1) * ncl, 0);
                sets.resize((s + 1) * ncl);
                eof.resize(s + 1, LC_NONE_ENTRY);
                if (s == 0)
                    continue;
                const TState cur = states[s]; // copy: `states` grows
                max_threads = std::max<uint32_t>(max_threads, (uint32_t)cur.th.size());
                // end of input: the first thread that can take MATCH wins
                for (size_t i = 0; i < cur.th.size() && eof[s] == LC_NONE_ENTRY; ++i)
                    for (auto& cd : cand[cur.th[i].w]) {
                        if (cd.target >= 0 || !holds(cd.asserts, cur.pk, K_EDGE, -1))
                            continue;
                        std::vector<uint16_t> lst;
                        for (uint32_t t = 0; t < T; ++t) {
                            int r = cur.th[i].reg[t];
                            if (cd.saves >> t & 1)
                                lst.push_back((uint16_t)(t << 8 | LC_TDFA_SRC_POS));
                            else if (r < 0)
                                lst.push_back((uint16_t)(t << 8 | LC_TDFA_SRC_UNSET));
                            else if ((uint32_t)r != t)
                                lst.push_back((uint16_t)(t << 8 | (uint32_t)r));
                        }
                        eof[s] = op_list(lst);
                        break;
                    }
                for (uint32_t c = 0; c < ncl && ok; ++c) {
                    const int nk = class_kind[c];
                    struct NT {
                        int w, parent;
                        uint64_t saves;
                    };
                    std::vector<NT> nts;
                    std::vector<char> taken(nw, 0);
                    for (size_t i = 0; i < cur.th.size(); ++i)
                        for (auto& cd : cand[cur.th[i].w]) {
                            if (cd.target < 0 || taken[cd.target])
                                continue;
                            if (cd.asserts && !holds(cd.asserts, cur.pk, nk, (int)c))
                                continue;
                            if (!walker_has(cd.target, (int)c))
                                continue;
                            taken[cd.target] = 1;
                            nts.push_back({cd.target, (int)i, cd.saves});
                        }
                    if (nts.empty())
                        continue;
                    if (nts.size() > 64) {
                        ok = false;
                        break;
                    }
                    // registers still referenced by inherited values
                    std::vector<char> used(256, 0);
                    uint64_t set_tags = 0;
                    for (auto& nt : nts) {
                        set_tags |= nt.saves;
                        for (uint32_t t = 0; t < T; ++t)
                            if (!(nt.saves >> t & 1)) {
                                int r = cur.th[nt.parent].reg[t];
                                if (r >= 0)
                                    used[r] = 1;
                            }
                    }
                    std::vector<int16_t> alloc(T, (int16_t)-1);
                    std::vector<uint8_t> setregs;
                    for (uint32_t t = 0; t < T; ++t)
                        if (set_tags >> t & 1) {
                            uint32_t r = t;
                            if (used[r]) {
                                r = T;
                                while (r < 255 && used[r])
                                    ++r;
                            }
                            if (r >= LC_TDFA_MAX_REGS) {
                                ok = false;
                                break;
                            }
                            used[r] = 1;
                            alloc[t] = (int16_t)r;
                            setregs.push_back((uint8_t)r);
                            nregs = std::max(nregs, r + 1);
                        }
                    if (!ok)
                        break;
                    TState nx;
                    nx.pk = ctx_full ? nk : 0;
                    for (auto& nt : nts) {
                        TThread th;
                        th.w = nt.w;
                        th.reg = cur.th[nt.parent].reg;
                        for (uint32_t t = 0; t < T; ++t)
                            if (nt.saves >> t & 1)
                                th.reg[t] = alloc[t];
                        nx.th.push_back(std::move(th));
                    }
                    uint32_t to = intern(std::move(nx));
                    if (!ok)
                        break;
                    std::vector<uint16_t> lst;
                    for (uint8_t r : setregs)
                        lst.push_back((uint16_t)((uint32_t)r << 8 | LC_TDFA_SRC_POS));
                    uint32_t ol = op_list(lst);
                    t1[s * ncl + c] = to | (ol << 16);
                    sets[s * ncl + c] = setregs;
                }
            }
            if (!ok)
                return;
            const uint32_t ns = (uint32_t)states.size();
            LcTdfaHeader th;
            memset(&th, 0, sizeof th);
            th.magic = LC_TDFA_MAGIC;
            th.ngroups = res.ngroups;
            th.nstates = ns;
            th.ncls = ncl;
            th.nregs = nregs;
            th.start = 1;
            th.row_bytes = (uint32_t)row_bytes;
            th.max_threads = max_threads;
            // row ns = the slow-path sink: entries whose steps set several registers lead there and it absorbs
            // every byte pair, so a kernel can test for it once per 16-byte chunk and redo that chunk step by step
            th.sink = ns;
            const size_t rw = (size_t)row_bytes / 4; // words per row
            std::vector<uint32_t> t2((size_t)(ns + 1) * rw, 0);
            for (uint32_t k = 0; k < ncl * ncl; ++k)
                t2[(size_t)ns * rw + k] = ns * (uint32_t)row_bytes | LC_TDFA_SLOW;
            for (uint32_t s = 1; s < ns; ++s)
                for (uint32_t c0 = 0; c0 < ncl; ++c0) {
                    uint32_t s1 = t1[(size_t)s * ncl + c0] & 0xFFFFu;
                    if (!s1)
                        continue;
                    const auto& A = sets[(size_t)s * ncl + c0];
                    for (uint32_t c1 = 0; c1 < ncl; ++c1) {
                        uint32_t s2 = t1[(size_t)s1 * ncl + c1] & 0xFFFFu;
                        if (!s2)
                            continue;
                        const auto& B = sets[(size_t)s1 * ncl + c1];
                        uint32_t e = s2 * (uint32_t)row_bytes;
                        if (A.size() > 1 || B.size() > 1) {
                            e = ns * (uint32_t)row_bytes | LC_TDFA_SLOW;
                            th.has_slow = 1;
                        } else {
                            if (!A.empty())
                                e |= (2u * A[0] + 2u) << 16;
                            if (!B.empty())
                                e |= (2u * B[0] + 2u) << 24;
                        }
                        t2[(size_t)s * rw + c0 * ncl + c1] = e;
                    }
                }
            std::vector<uint8_t> cls(byte_class, byte_class + 256);
            // run skipping: states whose every byte but at most two loops back without an op (state 0 = dead: always)
            std::vector<uint32_t> skip(ns + 1, 0);
            for (uint32_t s = 0; s < ns; ++s) {
                uint32_t nexit = 0, ex[2] = {0, 0};
                for (uint32_t b = 0; b < 256 && nexit <= 2; ++b) {
                    const uint32_t e = s ? t1[(size_t)s * ncl + byte_class[b]] : 0u;
                    if (e != s) { // another state, or ops on the way
                        if (nexit < 2)
                            ex[nexit] = b;
                        ++nexit;
                    }
                }
                if (nexit == 1)
                    ex[1] = ex[0]; // the exit test always checks both slots
                if (nexit <= 2)
                    skip[s] = LC_TDFA_SKIP | nexit << 16 | ex[1] << 8 | ex[0];
            }
            std::vector<uint8_t> tb(sizeof th, 0);
            put(tb, th.off_cls, cls);
            put(tb, th.off_t2, t2);
            put(tb, th.off_t1, t1);
            put(tb, th.off_eof, eof);
            put(tb, th.off_ops, ops);
            put(tb, th.off_skip, skip);
            while (tb.size() % 16)
                tb.push_back(0);
            th.total_bytes = (uint32_t)tb.size();
            memcpy(tb.data(), &th, sizeof th);
            if (tb.size() <= max_table_bytes)
                res.tdfa_blob.swap(tb);
        }();
    } catch (const Invalid& e) {
        res.valid = false;
        res.supported = false;
        res.error = std::string("invalid regex: ") + e.what();
    } catch (const Unsupported& e) {
        res.valid = true; // boost accepts it; this engine's automaton subset does not
        res.supported = false;
        res.error = std::string("unsupported regex: ") + e.what();
    }
    return res;
}

} // namespace lcb200
