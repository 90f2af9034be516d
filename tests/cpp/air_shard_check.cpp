// Host execution of the row-sharded constraint-program quotient (plonky3_b200/csrc/air_program.cu air_program_quotient_sharded_kernel):
// the same air_row_quotient over every rank's chunk-major row block, addressed as the kernel addresses it — the unit table
// (AirShardRow) and the owner arithmetic (air_shard_locate, air_shard_next_rank) of air_program.cuh — compiled as plain C++.  Reads
// jobs from stdin:
//
//   field width n_public n_nodes n_constraints  <nodes: op a b imm ...>  <constraints>  log_q log_n world
//     n_segments <segments: first column, end column, element offset (of a block of R = 2^log_q / world rows)>
//     <2^log_q x width LDE rows, bit-reversed>  <public values>  <alpha: 4 words>
//
// and answers each with one line "rc misplaced" (misplaced: the rows whose memory row or next row was not where the owner helpers
// put it), followed by one line per rank of R x 4 quotient words (Montgomery), entry m at natural index bitrev(rank R + m).
#include <cstdint>
#include <cstdio>
#include <iostream>
#include <vector>
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
#include "../../plonky3_b200/csrc/air_program.cuh"
using namespace p3;

template <int F> struct ShardEnv {
    const AirProgram *p;
    const std::vector<u32> *pubs, *zh_t, *izh_t;
    const std::vector<uint4> *ap;
    const u64 *units;
    const u32 *own, *peer;      // my block; the block of air_shard_next_rank(rank)
    u32 rank, peer_rank;
    unsigned log_rows, q;
    size_t misplaced = 0;
    std::vector<u32> slots;
    AirShardRow cur{}, nxt{};
    AirInsn insn(u32 pc) const { return p->insns[pc]; }
    u32 &slot(u32 s) { return slots[s]; }
    void set_rows(u32 m, u32 mn) {
        const AirShardLoc a = air_shard_locate(m, log_rows), b = air_shard_locate(mn, log_rows);
        misplaced += a.rank != rank || ((p->uses & AIR_USES_NEXT) && b.rank != peer_rank);
        cur = AirShardRow{own, units, a.row};
        nxt = AirShardRow{peer, units, b.row};
    }
    u32 local(u32 c) const { return cur.ld(c); }
    u32 next(u32 c) const { return nxt.ld(c); }
    u32 pub(u32 k) const { return (*pubs)[k]; }
    uint4 apow(u32 k) const { return (*ap)[k]; }
    u32 zh(u32 i) const { return (*zh_t)[i & ((1u << q) - 1u)]; }
    u32 inv_zh(u32 i) const { return (*izh_t)[i & ((1u << q) - 1u)]; }
};

template <int F>
static void quotient(const AirProgram &p, unsigned log_q, unsigned log_n, unsigned world, const std::vector<size_t> &segs,
                     const std::vector<u32> &lde, const std::vector<u32> &pubs, const u32 alpha[4]) {
    std::vector<u32> zh, izh;
    const AirDomain d = air_domain<F>(log_q, log_n, p.uses, zh, izh);
    const std::vector<uint4> ap = air_alpha_table<F>(alpha, p.n_constraints);
    unsigned log_g = 0;
    while ((1u << log_g) < world) log_g++;
    const unsigned log_rows = log_q - log_g;
    const size_t R = (size_t)1 << log_rows, W = p.width;
    // the unit table (air_shard_units) and every rank's chunk-major block, from the segment list
    std::vector<u64> units((W + AIR_UNIT - 1) / AIR_UNIT, 0);
    for (size_t s = 0; s < segs.size(); s += 3)
        for (size_t u = segs[s] / AIR_UNIT; u * AIR_UNIT < segs[s + 1]; u++) units[u] = air_unit_entry(segs[s + 2] - segs[s], segs[s + 1] - segs[s]);
    std::vector<std::vector<u32>> blocks(world, std::vector<u32>(R * W, 0xffffffffu));
    for (unsigned g = 0; g < world; g++)
        for (size_t s = 0; s < segs.size(); s += 3) {
            const size_t c0 = segs[s], c1 = segs[s + 1], off = segs[s + 2];
            for (size_t m = 0; m < R; m++)
                for (size_t c = c0; c < c1; c++) blocks[g][off + m * (c1 - c0) + (c - c0)] = lde[(g * R + m) * W + c];
        }
    size_t misplaced = 0;
    std::vector<std::vector<uint4>> out(world);
    for (unsigned g = 0; g < world; g++) {
        ShardEnv<F> env;
        env.p = &p; env.pubs = &pubs; env.zh_t = &zh; env.izh_t = &izh; env.ap = &ap; env.units = units.data();
        env.rank = g; env.peer_rank = air_shard_next_rank(g, log_g, d.q);
        env.own = blocks[g].data(); env.peer = blocks[env.peer_rank].data();
        env.log_rows = log_rows; env.q = d.q;
        env.slots.assign(p.n_slots + 1, 0xffffffffu);
        for (u32 m = 0; m < R; m++) out[g].push_back(air_row_quotient<F>(env, d, (u32)p.insns.size(), air_bitrev(g * (u32)R + m, log_q)));
        misplaced += env.misplaced;
    }
    printf("0 %zu\n", misplaced);
    for (auto &o : out) {
        for (auto &r : o) printf("%u %u %u %u ", r.x, r.y, r.z, r.w);
        printf("\n");
    }
}

int main() {
    int field;
    while (std::cin >> field) {
        uint32_t width, n_public;
        size_t n_nodes, n_cons, n_segs;
        std::cin >> width >> n_public >> n_nodes >> n_cons;
        std::vector<p3gpu_air_node> nodes(n_nodes);
        for (auto &n : nodes) std::cin >> n.op >> n.a >> n.b >> n.imm;
        std::vector<uint32_t> cons(n_cons);
        for (auto &c : cons) std::cin >> c;
        unsigned log_q, log_n, world;
        std::cin >> log_q >> log_n >> world >> n_segs;
        std::vector<size_t> segs(3 * n_segs);
        for (auto &s : segs) std::cin >> s;
        std::vector<u32> lde(((size_t)1 << log_q) * width), pubs(n_public);
        for (auto &v : lde) std::cin >> v;
        for (auto &v : pubs) std::cin >> v;
        u32 alpha[4];
        for (auto &v : alpha) std::cin >> v;
        AirProgram p;
        std::string err;
        const int32_t rc = air_compile(field, nodes.data(), n_nodes, cons.data(), n_cons, width, n_public, p, err);
        if (rc != P3GPU_OK) {
            printf("%d 0\n", rc);
            fprintf(stderr, "%s\n", err.c_str());
        } else if (field == BABY_BEAR) {
            quotient<BABY_BEAR>(p, log_q, log_n, world, segs, lde, pubs, alpha);
        } else {
            quotient<KOALA_BEAR>(p, log_q, log_n, world, segs, lde, pubs, alpha);
        }
        fflush(stdout);
    }
    return 0;
}
