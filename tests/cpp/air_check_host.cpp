// Host execution of the debug constraint check of plonky3_b200/csrc/air_program.cuh — the compiler under the check limits and
// air_row_check, which air_check.cu's kernel runs on every row — compiled as plain C++ (g++ ignores the CUDA function attributes).
// Reads jobs from stdin:
//
//   C field width n_public pre_width n_periodic n_nodes n_constraints  <nodes: op a b imm ...>  <constraints>
//       compile a check program (AIR_CHECK_LIMITS)
//   P ... as C                                                                  compile a quotient program (the default limits)
//   R ... as C, then  height  <height x width trace rows>  <height x pre_width preprocessed rows>  periodic_rows
//       <periodic_rows x n_periodic periodic table, row-major>  <public values>     check every row
//
// and answers each with one line "rc instructions slots" (the compiler's message on stderr), followed for `R` jobs by one line of
// "row constraint" pairs, one per failing constraint, rows ascending and each row's constraints in the order air_row_check reports
// them.
#include <cstdint>
#include <cstdio>
#include <iostream>
#include <vector>
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
#include "../../plonky3_b200/csrc/air_program.cuh"
using namespace p3;

struct HostCheckEnv {
    const AirProgram *p;
    const std::vector<u32> *trace, *pre, *per, *pubs;
    std::vector<u32> slots;
    size_t row = 0, nrow = 0, prow = 0, pnrow = 0, perow = 0;
    AirInsn insn(u32 pc) const { return p->insns[pc]; }
    u32 &slot(u32 s) { return slots[s]; }
    void set_rows(u32 i, u32 in) { row = (size_t)i * p->width; nrow = (size_t)in * p->width; }
    void set_ext_rows(u32 i, u32 in, u32 pr) { prow = (size_t)i * p->pre_width; pnrow = (size_t)in * p->pre_width; perow = (size_t)pr * p->n_periodic; }
    u32 local(u32 c) const { return (*trace)[row + c]; }
    u32 next(u32 c) const { return (*trace)[nrow + c]; }
    u32 pre_local(u32 c) const { return (*pre)[prow + c]; }
    u32 pre_next(u32 c) const { return (*pre)[pnrow + c]; }
    u32 periodic(u32 k) const { return (*per)[perow + k]; }
    u32 pub(u32 k) const { return (*pubs)[k]; }
};

template <int F> static void check_rows(const AirProgram &p, u32 height, const std::vector<u32> &trace, const std::vector<u32> &pre,
                                        const std::vector<u32> &per, u32 periodic_rows, const std::vector<u32> &pubs) {
    HostCheckEnv env;
    env.p = &p; env.trace = &trace; env.pre = &pre; env.per = &per; env.pubs = &pubs;
    env.slots.assign(p.n_slots + 1, 0xffffffffu);
    for (u32 i = 0; i < height; i++) {
        auto report = [&](u32 k) { printf("%u %u ", i, k); };
        air_row_check<F>(env, (u32)p.insns.size(), i, height, periodic_rows, report);
    }
    printf("\n");
}

int main() {
    std::string mode;
    while (std::cin >> mode) {
        int field;
        uint32_t width, n_public, pre_width, n_periodic;
        size_t n_nodes, n_cons;
        std::cin >> field >> width >> n_public >> pre_width >> n_periodic >> n_nodes >> n_cons;
        std::vector<p3gpu_air_node> nodes(n_nodes);
        for (auto &n : nodes) std::cin >> n.op >> n.a >> n.b >> n.imm;
        std::vector<uint32_t> cons(n_cons);
        for (auto &c : cons) std::cin >> c;
        AirProgram p;
        std::string err;
        const int32_t rc = mode == "P" ? air_compile(field, nodes.data(), n_nodes, cons.data(), n_cons, width, n_public, pre_width, n_periodic, p, err)
                                       : air_compile(field, nodes.data(), n_nodes, cons.data(), n_cons, width, n_public, pre_width, n_periodic, p, err,
                                                     AIR_CHECK_LIMITS);
        if (rc != P3GPU_OK) {
            printf("%d 0 0\n", rc);
            fprintf(stderr, "%s\n", err.c_str());
        } else {
            printf("%d %zu %u\n", rc, p.insns.size(), p.n_slots);
        }
        if (mode == "R") {
            u32 height, periodic_rows;
            std::cin >> height;
            std::vector<u32> trace((size_t)height * width), pre((size_t)height * pre_width), pubs(n_public);
            for (auto &v : trace) std::cin >> v;
            for (auto &v : pre) std::cin >> v;
            std::cin >> periodic_rows;
            std::vector<u32> per((size_t)periodic_rows * n_periodic);
            for (auto &v : per) std::cin >> v;
            for (auto &v : pubs) std::cin >> v;
            if (rc != P3GPU_OK) { printf("\n"); continue; }
            if (field == BABY_BEAR) check_rows<BABY_BEAR>(p, height, trace, pre, per, periodic_rows, pubs);
            else check_rows<KOALA_BEAR>(p, height, trace, pre, per, periodic_rows, pubs);
        }
        fflush(stdout);
    }
    return 0;
}
