// Host execution of plonky3_b200/csrc/air_program.cuh for programs with preprocessed and periodic columns — the layout compiler and
// the EXT instance of air_row_quotient the device kernel runs for them — compiled as plain C++ (g++ ignores the CUDA function
// attributes).  The companion of tests/cpp/air_program_check.cpp.  Reads jobs from stdin:
//
//   L field width n_public pre_width n_periodic n_nodes n_constraints  <nodes: op a b imm ...>  <constraints>
//   Q field width n_public pre_width n_periodic n_nodes n_constraints  <nodes> <constraints>  log_q log_n
//     <2^log_q x width LDE prefix rows, bit-reversed>  <2^log_q x pre_width preprocessed LDE prefix rows, bit-reversed>
//     log_periodic_rows  <2^log_periodic_rows x n_periodic periodic table, row-major>  <public values> <alpha: 4 words>
//
// and answers each with one line "rc instructions slots max_live" (max_live: the most values live at once in the emitted stream,
// recomputed here from the instructions), followed for `Q` jobs by a line of 2^log_q x 4 quotient words (Montgomery).
#include <cstdint>
#include <cstdio>
#include <iostream>
#include <vector>
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
#include "../../plonky3_b200/csrc/air_program.cuh"
using namespace p3;

template <int F> struct HostEnv {
    const AirProgram *p;
    const std::vector<u32> *lde, *pre, *per, *pubs, *zh_t, *izh_t;
    const std::vector<uint4> *ap;
    std::vector<u32> slots;
    size_t row = 0, nrow = 0, prow = 0, pnrow = 0, perow = 0;
    unsigned q = 0;
    AirInsn insn(u32 pc) const { return p->insns[pc]; }
    u32 &slot(u32 s) { return slots[s]; }
    void set_rows(u32 m, u32 mn) { row = (size_t)m * p->width; nrow = (size_t)mn * p->width; }
    void set_ext_rows(u32 m, u32 mn, u32 pr) { prow = (size_t)m * p->pre_width; pnrow = (size_t)mn * p->pre_width; perow = (size_t)pr * p->n_periodic; }
    u32 local(u32 c) const { return (*lde)[row + c]; }
    u32 next(u32 c) const { return (*lde)[nrow + c]; }
    u32 pre_local(u32 c) const { return (*pre)[prow + c]; }
    u32 pre_next(u32 c) const { return (*pre)[pnrow + c]; }
    u32 periodic(u32 k) const { return (*per)[perow + k]; }
    u32 pub(u32 k) const { return (*pubs)[k]; }
    uint4 apow(u32 k) const { return (*ap)[k]; }
    u32 zh(u32 i) const { return (*zh_t)[i & ((1u << q) - 1u)]; }
    u32 inv_zh(u32 i) const { return (*izh_t)[i & ((1u << q) - 1u)]; }
};

static size_t max_live(const AirProgram &p) {
    // value written at instruction w into slot s is live until its last read before the next write of s
    std::vector<long> written(p.n_slots + 1, -1), last_read(p.n_slots + 1, -1);
    std::vector<std::pair<long, long>> iv;
    auto close = [&](u32 s) { if (written[s] >= 0) iv.push_back({written[s], last_read[s]}); };
    for (size_t pc = 0; pc < p.insns.size(); pc++) {
        const u32 op = p.insns[pc].op_dst & 15u, dst = p.insns[pc].op_dst >> 4, arg = p.insns[pc].arg;
        if (op == P3GPU_AIR_ADD || op == P3GPU_AIR_SUB || op == P3GPU_AIR_MUL) { last_read[arg & 0xffff] = pc; last_read[arg >> 16] = pc; }
        else if (op == P3GPU_AIR_NEG || op == AIR_OP_FOLD) last_read[arg] = pc;
        if (op == AIR_OP_FOLD) continue;
        close(dst);
        written[dst] = (long)pc; last_read[dst] = -1;
    }
    for (u32 s = 0; s < p.n_slots; s++) close(s);
    size_t best = 0;
    for (size_t pc = 0; pc < p.insns.size(); pc++) {
        size_t n = 0;
        for (auto &v : iv) n += v.first <= (long)pc && v.second > (long)pc;
        best = std::max(best, n);
    }
    return best;
}

template <int F> static void quotient(const AirProgram &p, unsigned log_q, unsigned log_n, const std::vector<u32> &lde, const std::vector<u32> &pre,
                                      const std::vector<u32> &per, unsigned log_periodic_rows, const std::vector<u32> &pubs, const u32 alpha[4]) {
    std::vector<u32> zh, izh;
    AirDomain d = air_domain<F>(log_q, log_n, p.uses, zh, izh);
    d.periodic_mask = (1u << log_periodic_rows) - 1u;
    const std::vector<uint4> ap = air_alpha_table<F>(alpha, p.n_constraints);
    HostEnv<F> env;
    env.p = &p; env.lde = &lde; env.pre = &pre; env.per = &per; env.pubs = &pubs; env.zh_t = &zh; env.izh_t = &izh; env.ap = &ap; env.q = d.q;
    env.slots.assign(p.n_slots + 1, 0xffffffffu);
    for (u32 i = 0; i < (1u << log_q); i++) {
        const uint4 r = air_row_quotient<F, true>(env, d, (u32)p.insns.size(), i);
        printf("%u %u %u %u ", r.x, r.y, r.z, r.w);
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
        const int32_t rc = air_compile(field, nodes.data(), n_nodes, cons.data(), n_cons, width, n_public, pre_width, n_periodic, p, err);
        if (rc != P3GPU_OK) {
            printf("%d 0 0 0\n", rc);
            fprintf(stderr, "%s\n", err.c_str());
        } else {
            printf("%d %zu %u %zu\n", rc, p.insns.size(), p.n_slots, max_live(p));
        }
        if (mode == "Q") {
            unsigned log_q, log_n, log_per;
            std::cin >> log_q >> log_n;
            std::vector<u32> lde(((size_t)1 << log_q) * width), pre(((size_t)1 << log_q) * pre_width), pubs(n_public);
            for (auto &v : lde) std::cin >> v;
            for (auto &v : pre) std::cin >> v;
            std::cin >> log_per;
            std::vector<u32> per(((size_t)1 << log_per) * n_periodic);
            for (auto &v : per) std::cin >> v;
            for (auto &v : pubs) std::cin >> v;
            u32 alpha[4];
            for (auto &v : alpha) std::cin >> v;
            if (rc != P3GPU_OK) { printf("\n"); continue; }
            if (field == BABY_BEAR) quotient<BABY_BEAR>(p, log_q, log_n, lde, pre, per, log_per, pubs, alpha);
            else quotient<KOALA_BEAR>(p, log_q, log_n, lde, pre, per, log_per, pubs, alpha);
        }
        fflush(stdout);
    }
    return 0;
}
