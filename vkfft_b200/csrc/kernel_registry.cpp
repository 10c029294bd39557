#include "kernel_registry.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {
std::vector<b2_kernel_info*>& table() {
    static std::vector<b2_kernel_info*> t;
    return t;
}
// B200FFT_VARIANTS="kind:prec:n=variant,..." (tuning / experiments); unset -> variant 0 everywhere
int variant_override(int kind, int prec, int n) {
    const char* e = getenv("B200FFT_VARIANTS");
    if (!e) return 0;
    for (const char* p = e; *p;) {
        int k, pr, nn, v, used = 0;
        if (sscanf(p, "%d:%d:%d=%d%n", &k, &pr, &nn, &v, &used) == 4) {
            if (k == kind && pr == prec && nn == n) return v;
            p += used;
        } else {
            break;
        }
        if (*p == ',') ++p;
    }
    return 0;
}
}  // namespace

extern "C" void b2_register_kernel(const b2_kernel_info* k) {
    b2_kernel_info* m = const_cast<b2_kernel_info*>(k);
    int v = 0;
    for (const b2_kernel_info* o : table())
        if (o->kind == k->kind && o->prec == k->prec && o->n == k->n && o->inv == k->inv && o->ops == k->ops) ++v;
    m->variant = v;
    table().push_back(m);
}
namespace { b2_kernel_provider g_provider = nullptr; }
extern "C" void b2_set_kernel_provider(b2_kernel_provider p) { g_provider = p; }
extern "C" const b2_kernel_info* b2_find_kernel_variant(int kind, int prec, int n, int inv, int ops, int variant) {
    for (const b2_kernel_info* k : table())
        if (k->kind == kind && k->prec == prec && k->n == n && k->inv == inv && k->ops == ops && k->variant == variant)
            return k;
    if (variant == 0 && g_provider) return g_provider(kind, prec, n, inv, ops);
    return nullptr;
}
extern "C" const b2_kernel_info* b2_find_kernel(int kind, int prec, int n, int inv, int ops) {
    const int v = variant_override(kind, prec, n);
    const b2_kernel_info* k = v ? b2_find_kernel_variant(kind, prec, n, inv, ops, v) : nullptr;
    return k ? k : b2_find_kernel_variant(kind, prec, n, inv, ops, 0);
}
extern "C" int b2_kernel_count(void) { return (int)table().size(); }
extern "C" const b2_kernel_info* b2_kernel_at(int i) { return table()[i]; }

// ---- fused Four-Step kernels ---------------------------------------------------------------------------------------
namespace {
std::vector<b2_fused_info*>& ftable() {
    static std::vector<b2_fused_info*> t;
    return t;
}
}  // namespace
extern "C" void b2_register_fused(const b2_fused_info* k) {
    b2_fused_info* m = const_cast<b2_fused_info*>(k);
    int v = 0;
    for (const b2_fused_info* o : ftable())
        if (o->prec == k->prec && o->n1 == k->n1 && o->n2 == k->n2 && o->inv == k->inv) ++v;
    m->variant = v;
    ftable().push_back(m);
}
extern "C" const b2_fused_info* b2_find_fused_variant(int prec, int n1, int n2, int inv, int variant) {
    for (const b2_fused_info* k : ftable())
        if (k->prec == prec && k->n1 == n1 && k->n2 == n2 && k->inv == inv && k->variant == variant) return k;
    return nullptr;
}
// B200FFT_FUSED_VARIANTS="n1xn2=variant,..." selects a non-default CTA shape (tuning)
extern "C" const b2_fused_info* b2_find_fused(int prec, int n1, int n2, int inv) {
    int v = 0;
    if (const char* e = getenv("B200FFT_FUSED_VARIANTS")) {
        for (const char* p = e; *p;) {
            int a, b, vv, used = 0;
            if (sscanf(p, "%dx%d=%d%n", &a, &b, &vv, &used) == 3) {
                if (a == n1 && b == n2) v = vv;
                p += used;
            } else break;
            if (*p == ',') ++p;
        }
    }
    const b2_fused_info* k = v ? b2_find_fused_variant(prec, n1, n2, inv, v) : nullptr;
    return k ? k : b2_find_fused_variant(prec, n1, n2, inv, 0);
}
extern "C" int b2_fused_count(void) { return (int)ftable().size(); }
extern "C" const b2_fused_info* b2_fused_at(int i) { return ftable()[i]; }

// ---- cluster Four-Step kernels ---------------------------------------------------------------------------------------
namespace {
std::vector<b2_cluster_info*>& ctable() {
    static std::vector<b2_cluster_info*> t;
    return t;
}
}  // namespace
extern "C" void b2_register_cluster(const b2_cluster_info* k) {
    b2_cluster_info* m = const_cast<b2_cluster_info*>(k);
    int v = 0;
    for (const b2_cluster_info* o : ctable())
        if (o->prec == k->prec && o->n1 == k->n1 && o->n2 == k->n2 && o->inv == k->inv) ++v;
    m->variant = v;
    ctable().push_back(m);
}
// B200FFT_CLUSTER4_VARIANTS="n1xn2=variant,..." selects a non-default cluster shape (A/B timing)
extern "C" const b2_cluster_info* b2_find_cluster(int prec, int n1, int n2, int inv) {
    int v = 0;
    if (const char* e = getenv("B200FFT_CLUSTER4_VARIANTS")) {
        for (const char* p = e; *p;) {
            int a, b, vv, used = 0;
            if (sscanf(p, "%dx%d=%d%n", &a, &b, &vv, &used) == 3) {
                if (a == n1 && b == n2) v = vv;
                p += used;
            } else break;
            if (*p == ',') ++p;
        }
    }
    const b2_cluster_info* dflt = nullptr;
    for (const b2_cluster_info* k : ctable()) {
        if (k->prec != prec || k->n1 != n1 || k->n2 != n2 || k->inv != inv) continue;
        if (k->variant == v) return k;
        if (k->variant == 0) dflt = k;
    }
    return dflt;
}
extern "C" int b2_cluster_count(void) { return (int)ctable().size(); }
extern "C" const b2_cluster_info* b2_cluster_at(int i) { return ctable()[i]; }
