// yk_dict.cpp -- label / taint dictionary encoder (host C++; see include/ykgpu_dict.h for what it restates).
#include "../../include/ykgpu_dict.h"
#include "../../include/ykgpu.h"

#include <algorithm>
#include <cerrno>
#include <cstdlib>
#include <cstring>
#include <map>
#include <new>
#include <string>
#include <vector>

namespace {

constexpr int LABEL_BITS = 63;               // bit 63 = impossible
constexpr uint64_t IMPOSSIBLE = 1ull << 63;
constexpr int TAINT_BITS = 64;
const char* UNSCHED_KEY = "node.kubernetes.io/unschedulable";

bool is_alnum(char c) { return (c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9'); }
bool name_chars(const std::string& s) {   // ([A-Za-z0-9][-A-Za-z0-9_.]*)?[A-Za-z0-9]
    if (s.empty() || !is_alnum(s.front()) || !is_alnum(s.back())) return false;
    for (char c : s) if (!is_alnum(c) && c != '-' && c != '_' && c != '.') return false;
    return true;
}
// k8s.io/apimachinery validation.IsValidLabelValue
bool valid_label_value(const std::string& v) { return v.size() <= 63 && (v.empty() || name_chars(v)); }
// validation.IsQualifiedName: [dns-subdomain "/"] name
bool valid_label_key(const std::string& k) {
    std::string name = k;
    size_t slash = k.find('/');
    if (slash != std::string::npos) {
        if (k.find('/', slash + 1) != std::string::npos) return false;
        std::string prefix = k.substr(0, slash);
        name = k.substr(slash + 1);
        if (prefix.empty() || prefix.size() > 253) return false;
        for (char c : prefix) if (!((c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '-' || c == '.')) return false;
        if (!is_alnum(prefix.front()) || !is_alnum(prefix.back())) return false;
    }
    return !name.empty() && name.size() <= 63 && name_chars(name);
}
bool parse_i64(const std::string& s, int64_t* out) {   // strconv.ParseInt(s, 10, 64)
    if (s.empty()) return false;
    errno = 0;
    char* end = nullptr;
    long long v = strtoll(s.c_str(), &end, 10);
    if (errno != 0 || *end != '\0') return false;
    if (s[0] == ' ' || s[0] == '\t') return false;
    *out = v;
    return true;
}

struct Req {
    std::string key;
    uint32_t op = 0;
    std::vector<std::string> values;   // sorted, unique
    int64_t num = 0;
    bool valid = true;                 // labels.NewRequirement accepted it
};

Req parse_req(const yk_requirement& r) {
    Req q;
    q.key = r.key ? r.key : "";
    q.op = r.op;
    for (uint32_t i = 0; i < r.n_values; ++i) q.values.emplace_back(r.values[i] ? r.values[i] : "");
    q.valid = valid_label_key(q.key);
    switch (r.op) {
        case YK_OP_IN: case YK_OP_NOT_IN: if (q.values.empty()) q.valid = false; break;
        case YK_OP_EXISTS: case YK_OP_DOES_NOT_EXIST: if (!q.values.empty()) q.valid = false; break;
        case YK_OP_GT: case YK_OP_LT:
            if (q.values.size() != 1 || !parse_i64(q.values[0], &q.num)) q.valid = false;
            break;
        default: q.valid = false;
    }
    for (const auto& v : q.values) if (!valid_label_value(v)) q.valid = false;
    std::sort(q.values.begin(), q.values.end());
    q.values.erase(std::unique(q.values.begin(), q.values.end()), q.values.end());
    return q;
}

using Labels = std::map<std::string, std::string>;

// labels.Requirement.Matches for the POSITIVE form of the operator
bool match_positive(const Req& q, uint32_t op, const Labels& l) {
    auto it = l.find(q.key);
    switch (op) {
        case YK_OP_IN: return it != l.end() && std::binary_search(q.values.begin(), q.values.end(), it->second);
        case YK_OP_EXISTS: return it != l.end();
        case YK_OP_GT: case YK_OP_LT: {
            int64_t v;
            if (it == l.end() || !parse_i64(it->second, &v)) return false;
            return op == YK_OP_GT ? v > q.num : v < q.num;
        }
        default: return false;
    }
}
bool match_req(const Req& q, const Labels& l) {
    switch (q.op) {
        case YK_OP_NOT_IN: return !match_positive(q, YK_OP_IN, l);
        case YK_OP_DOES_NOT_EXIST: return !match_positive(q, YK_OP_EXISTS, l);
        default: return match_positive(q, q.op, l);
    }
}

struct Term {
    std::vector<Req> exprs;
    std::vector<Req> fields;
    bool parse_error = false;
};
Term parse_term(const yk_selector_term& t) {
    Term out;
    for (uint32_t i = 0; i < t.n_expressions; ++i) {
        out.exprs.push_back(parse_req(t.expressions[i]));
        if (!out.exprs.back().valid) out.parse_error = true;
    }
    for (uint32_t i = 0; i < t.n_fields; ++i) {   // nodeSelectorRequirementsAsFieldSelector: In / NotIn with one value
        const yk_requirement& r = t.fields[i];
        Req q;
        q.key = r.key ? r.key : "";
        q.op = r.op;
        for (uint32_t j = 0; j < r.n_values; ++j) q.values.emplace_back(r.values[j] ? r.values[j] : "");
        if ((r.op != YK_OP_IN && r.op != YK_OP_NOT_IN) || q.values.size() != 1) { q.valid = false; out.parse_error = true; }
        out.fields.push_back(q);
    }
    return out;
}
bool match_term(const Term& t, const Labels& l, const std::string& node_name) {
    if (t.parse_error) return false;
    for (const Req& q : t.exprs) if (!match_req(q, l)) return false;
    for (const Req& q : t.fields) {
        const std::string have = q.key == "metadata.name" ? node_name : std::string();
        const bool eq = have == q.values[0];
        if (q.op == YK_OP_IN ? !eq : eq) return false;
    }
    return true;
}

struct Expr {            // one dictionary entry = one label bit
    bool whole = false;  // false: single positive requirement; true: OR of terms
    Req req; uint32_t pos_op = 0;
    std::vector<Term> terms;
};
bool eval_expr(const Expr& e, const Labels& l, const std::string& name) {
    if (!e.whole) return match_positive(e.req, e.pos_op, l);
    for (const Term& t : e.terms) if (match_term(t, l, name)) return true;
    return false;
}

std::string canon_req(const Req& q, uint32_t pos_op) {
    std::string s = "R\x1e" + q.key + "\x1e" + std::to_string(pos_op);
    if (pos_op == YK_OP_GT || pos_op == YK_OP_LT) s += "\x1e" + std::to_string(q.num);
    else for (const auto& v : q.values) s += "\x1e" + v;
    return s;
}
std::string canon_terms(const std::vector<Term>& ts) {
    std::string s = "S";
    for (const Term& t : ts) {
        s += "\x1dT";
        if (t.parse_error) { s += "!"; continue; }
        for (const Req& q : t.exprs) { s += "\x1d" + canon_req(q, q.op) + "#" + std::to_string(q.op); }
        for (const Req& q : t.fields) { s += "\x1d" "F" + q.key + "\x1e" + std::to_string(q.op) + "\x1e" + q.values[0]; }
    }
    return s;
}

struct TaintKey { std::string key, value; uint32_t effect; };

struct NodeRec {
    bool present = false;
    std::string name;
    Labels labels;
    std::vector<TaintKey> taints;
    bool unsched = false;
    uint64_t label_bits = 0, taint_bits = 0;
};

}  // namespace

struct yk_dict {
    std::vector<Expr> exprs;
    std::map<std::string, int> expr_index;
    std::vector<TaintKey> taints;
    std::map<std::string, int> taint_index;
    std::vector<NodeRec> nodes;
    std::map<std::string, uint32_t> by_name;
    uint64_t gen = 0;

    int label_bit(const std::string& canon, Expr&& e) {
        auto it = expr_index.find(canon);
        if (it != expr_index.end()) return it->second;
        if ((int)exprs.size() >= LABEL_BITS) return -1;
        int b = (int)exprs.size();
        exprs.push_back(std::move(e));
        expr_index.emplace(canon, b);
        for (NodeRec& n : nodes)   // existing nodes get the new bit evaluated
            if (n.present && eval_expr(exprs[(size_t)b], n.labels, n.name)) n.label_bits |= 1ull << b;
        ++gen;
        return b;
    }
    int taint_bit(const TaintKey& t, bool create) {
        std::string c = t.key + "\x1e" + t.value + "\x1e" + std::to_string(t.effect);
        auto it = taint_index.find(c);
        if (it != taint_index.end()) return it->second;
        if (!create || (int)taints.size() >= TAINT_BITS) return -1;
        int b = (int)taints.size();
        taints.push_back(t);
        taint_index.emplace(c, b);
        ++gen;   // pods with key-specific tolerations must be re-encoded
        return b;
    }
};

static bool tolerates(const yk_toleration& t, const TaintKey& x) {   // core/v1 Toleration.ToleratesTaint
    if (t.effect != YK_EFFECT_ALL && t.effect != x.effect) return false;
    const char* key = t.key ? t.key : "";
    if (key[0] && x.key != key) return false;
    if (t.op == YK_TOL_EXISTS) return true;
    if (t.op == YK_TOL_EQUAL) return x.value == (t.value ? t.value : "");
    return false;
}

extern "C" {

yk_dict* yk_dict_create(void) { return new (std::nothrow) yk_dict(); }
void yk_dict_destroy(yk_dict* d) { delete d; }
uint64_t yk_dict_generation(const yk_dict* d) { return d ? d->gen : 0; }

int yk_dict_node(yk_dict* d, uint32_t idx, const char* name, uint32_t n_labels, const char* const* keys,
                 const char* const* values, uint32_t n_taints, const yk_taint* taints, int32_t unschedulable,
                 uint64_t* label_bits, uint64_t* taint_bits) {
    if (!d || !name || (n_labels && (!keys || !values)) || (n_taints && !taints)) return YK_ERR_ARG;
    if (idx >= d->nodes.size()) d->nodes.resize((size_t)idx + 1);
    NodeRec& n = d->nodes[idx];
    if (n.present) d->by_name.erase(n.name);
    n = NodeRec();
    n.present = true;
    n.name = name;
    d->by_name[n.name] = idx;
    for (uint32_t i = 0; i < n_labels; ++i) n.labels[keys[i] ? keys[i] : ""] = values[i] ? values[i] : "";
    n.unsched = unschedulable != 0;
    int rc = YK_OK;
    auto add_taint = [&](const TaintKey& t) {
        if (t.effect != YK_EFFECT_NO_SCHEDULE && t.effect != YK_EFFECT_NO_EXECUTE) return;   // PreferNoSchedule is not a filter
        n.taints.push_back(t);
        int b = d->taint_bit(t, true);
        if (b < 0) rc = YK_ERR_RANGE;   // more than 64 distinct hard taints: cannot be represented, never approximated
        else n.taint_bits |= 1ull << b;
    };
    for (uint32_t i = 0; i < n_taints; ++i)
        add_taint(TaintKey{taints[i].key ? taints[i].key : "", taints[i].value ? taints[i].value : "", taints[i].effect});
    if (n.unsched) add_taint(TaintKey{UNSCHED_KEY, "", YK_EFFECT_NO_SCHEDULE});
    for (size_t b = 0; b < d->exprs.size(); ++b)
        if (eval_expr(d->exprs[b], n.labels, n.name)) n.label_bits |= 1ull << b;
    if (label_bits) *label_bits = n.label_bits;
    if (taint_bits) *taint_bits = n.taint_bits;
    return rc;
}

int yk_dict_node_remove(yk_dict* d, uint32_t idx) {
    if (!d || idx >= d->nodes.size() || !d->nodes[idx].present) return YK_ERR_ARG;
    d->by_name.erase(d->nodes[idx].name);
    d->nodes[idx] = NodeRec();
    return YK_OK;
}

int yk_dict_node_bits(const yk_dict* d, uint32_t idx, uint64_t* label_bits, uint64_t* taint_bits) {
    if (!d || idx >= d->nodes.size() || !d->nodes[idx].present) return YK_ERR_ARG;
    if (label_bits) *label_bits = d->nodes[idx].label_bits;
    if (taint_bits) *taint_bits = d->nodes[idx].taint_bits;
    return YK_OK;
}

}  // extern "C"

// yk_dict_pod (at == NULL) and yk_dict_pod_required_node (at = the required node's name): the required-affinity terms are
// resolved against `at` first -- a term whose matchFields reject it is dropped, one whose fields accept it keeps only its
// expressions, and one left with no expression matches unconditionally
static int encode_pod(yk_dict* d, const yk_pod_spec* pod, const char* at, yk_pod_masks* out) {
    uint64_t need = 0, deny = 0, tol = 0;
    uint32_t flags = 0, want_node = YK_NONE;
    auto need_bit = [&](int b) { if (b < 0) flags |= YK_ASK_SLOWPATH; else need |= 1ull << b; };
    auto deny_bit = [&](int b) { if (b < 0) flags |= YK_ASK_SLOWPATH; else deny |= 1ull << b; };
    auto positive_bit = [&](const Req& q, uint32_t pos_op) {
        Expr e; e.whole = false; e.req = q; e.pos_op = pos_op;
        return d->label_bit(canon_req(q, pos_op), std::move(e));
    };

    // pod.Spec.NodeSelector: labels.SelectorFromSet -- exact key=value, no validation
    for (uint32_t i = 0; i < pod->n_selector; ++i) {
        Req q;
        q.key = pod->selector_keys[i] ? pod->selector_keys[i] : "";
        q.op = YK_OP_IN;
        q.values.emplace_back(pod->selector_values[i] ? pod->selector_values[i] : "");
        need_bit(positive_bit(q, YK_OP_IN));
    }
    // required node affinity
    if (pod->has_required_affinity) {
        std::vector<Term> terms;
        bool always = false;
        for (uint32_t i = 0; i < pod->n_terms; ++i) {
            const yk_selector_term& t = pod->terms[i];
            if (t.n_expressions == 0 && t.n_fields == 0) continue;   // nil or empty term selects no objects
            Term pt = parse_term(t);
            if (at && !pt.fields.empty()) {
                bool accept = true;
                for (const Req& q : pt.fields) {
                    if (!q.valid) { accept = false; break; }
                    const bool eq = (q.key == "metadata.name" ? std::string(at) : std::string()) == q.values[0];
                    if (q.op == YK_OP_IN ? !eq : eq) accept = false;
                }
                if (!accept) continue;
                pt.fields.clear();
                pt.parse_error = false;
                for (const Req& q : pt.exprs) if (!q.valid) pt.parse_error = true;
                if (pt.exprs.empty()) always = true;
            }
            terms.push_back(std::move(pt));
        }
        if (always) {}                            // a term matches the node whatever its labels: no bit
        else if (terms.empty()) need |= IMPOSSIBLE;   // nil / empty term list matches nothing
        else if (terms.size() == 1 && terms[0].fields.empty()) {
            if (terms[0].parse_error) need |= IMPOSSIBLE;
            else for (const Req& q : terms[0].exprs) {
                switch (q.op) {
                    case YK_OP_IN: need_bit(positive_bit(q, YK_OP_IN)); break;
                    case YK_OP_NOT_IN: deny_bit(positive_bit(q, YK_OP_IN)); break;
                    case YK_OP_EXISTS: need_bit(positive_bit(q, YK_OP_EXISTS)); break;
                    case YK_OP_DOES_NOT_EXIST: deny_bit(positive_bit(q, YK_OP_EXISTS)); break;
                    default: need_bit(positive_bit(q, q.op)); break;   // Gt / Lt
                }
            }
        } else {
            Expr e; e.whole = true; e.terms = terms;
            need_bit(d->label_bit(canon_terms(terms), std::move(e)));
        }
    }
    // tolerations against every known hard taint
    bool tolerate_all = false;
    for (uint32_t i = 0; i < pod->n_tolerations; ++i) {
        const yk_toleration& t = pod->tolerations[i];
        if (t.op == YK_TOL_EXISTS && (!t.key || !t.key[0]) && t.effect == YK_EFFECT_ALL) tolerate_all = true;
    }
    if (tolerate_all) tol = ~0ull;   // also covers taints registered later
    else for (size_t b = 0; b < d->taints.size(); ++b)
        for (uint32_t i = 0; i < pod->n_tolerations; ++i)
            if (tolerates(pod->tolerations[i], d->taints[b])) { tol |= 1ull << b; break; }
    // pod.Spec.NodeName, and the required node
    if (at) {
        auto it = d->by_name.find(at);
        if (it == d->by_name.end()) need |= IMPOSSIBLE; else want_node = it->second;
        if (pod->node_name && pod->node_name[0] && std::strcmp(pod->node_name, at) != 0) need |= IMPOSSIBLE;
    } else if (pod->node_name && pod->node_name[0]) {
        auto it = d->by_name.find(pod->node_name);
        if (it == d->by_name.end()) need |= IMPOSSIBLE; else want_node = it->second;
    }
    out->tolerated_bits = tol; out->required_bits = need; out->forbidden_bits = deny;
    out->required_node = want_node; out->flags = flags;
    return YK_OK;
}

extern "C" {

int yk_dict_pod(yk_dict* d, const yk_pod_spec* pod, yk_pod_masks* out) {
    if (!d || !pod || !out) return YK_ERR_ARG;
    return encode_pod(d, pod, nullptr, out);
}

int yk_dict_pod_required_node(yk_dict* d, const yk_pod_spec* pod, const char* node_name, yk_pod_masks* out) {
    if (!d || !pod || !node_name || !out) return YK_ERR_ARG;
    return encode_pod(d, pod, node_name, out);
}

}  // extern "C"
