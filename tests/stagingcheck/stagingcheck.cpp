// Host-compiled shim over csrc/staging.h for tests/test_staging.py.  A carve is a list of takes (kind, element size, count);
// it runs on null bases, so every pointer a take returns is its offset.  No CUDA call is reached.
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "../../openvslam_b200/csrc/staging.h"

namespace {

char g_error[512];

struct Take { int kind, elem; size_t n; };   // kind: 0 in, 1 io, 2 out, 3 dev

struct B16 { unsigned char b[16]; };

template <typename T>
void take_as(ovs::Staging& S, int kind, size_t n, size_t* h_off, size_t* d_off) {
    T* host = nullptr;
    T* dev = nullptr;
    if (kind == 0) dev = S.in(host, n);
    else if (kind == 1) dev = S.io(host, n);
    else if (kind == 2) dev = S.out(host, n);
    else dev = S.dev<T>(n);
    *h_off = kind == 3 ? (size_t)-1 : reinterpret_cast<size_t>(host);
    *d_off = reinterpret_cast<size_t>(dev);
}

// h_off / d_off: the offsets of each take (h_off of a device take: -1); h_end: the host arena's size after each take
void run(ovs::Staging& S, const Take* t, int n, size_t* h_off, size_t* d_off, size_t* h_end) {
    for (int i = 0; i < n; ++i) {
        size_t ho, dof;
        switch (t[i].elem) {
            case 1: take_as<unsigned char>(S, t[i].kind, t[i].n, &ho, &dof); break;
            case 2: take_as<unsigned short>(S, t[i].kind, t[i].n, &ho, &dof); break;
            case 4: take_as<float>(S, t[i].kind, t[i].n, &ho, &dof); break;
            case 8: take_as<double>(S, t[i].kind, t[i].n, &ho, &dof); break;
            default: take_as<B16>(S, t[i].kind, t[i].n, &ho, &dof); break;
        }
        if (h_off) h_off[i] = ho;
        if (d_off) d_off[i] = dof;
        if (h_end) h_end[i] = S.h.off;
    }
}

}  // namespace

namespace ovs {
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}
}  // namespace ovs

extern "C" {

// One counting carve (n <= 64 takes).  summary: [0] ordered [1] upload end [2] download begin [3] host size, the download's
// end [4] device size
void sc_carve(const int* kind, const int* elem, const size_t* count, int n, size_t* h_off, size_t* d_off, size_t* h_end,
              size_t* summary) {
    Take t[64];
    for (int i = 0; i < n; ++i) t[i] = Take{kind[i], elem[i], count[i]};
    ovs::Staging S;
    run(S, t, n, h_off, d_off, h_end);
    summary[0] = S.ordered ? 1 : 0;
    summary[1] = S.io_end;
    summary[2] = S.down_begin();
    summary[3] = S.h.off;
    summary[4] = S.d.off;
}

// ovs::stage on empty arenas (n <= 64 takes).  Returns its code; *allocated: 1 when an arena was touched.
int sc_stage(const int* kind, const int* elem, const size_t* count, int n, int* allocated) {
    Take t[64];
    for (int i = 0; i < n; ++i) t[i] = Take{kind[i], elem[i], count[i]};
    uint8_t* h_base = nullptr; uint8_t* d_base = nullptr;
    size_t h_cap = 0, d_cap = 0;
    ovs::Staging S;
    g_error[0] = 0;
    const int rc = ovs::stage(S, h_base, h_cap, d_base, d_cap, [&](ovs::Staging& s) { run(s, t, n, nullptr, nullptr, nullptr); });
    *allocated = (h_base || d_base || h_cap || d_cap) ? 1 : 0;
    return rc;
}

const char* sc_error() { return g_error; }

}  // extern "C"
