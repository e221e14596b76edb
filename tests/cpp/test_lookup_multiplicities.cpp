// The m(X) column of the log-derivative lookup (mv_lookup::Argument::prepare): Ops::lookup_multiplicities, whose default body
// is the host index (first usable table row per value), against DeviceOps, which calls b200zk_lookup_multiplicities.
//   usage: test_lookup_multiplicities host <in.bin> <out.bin>     the host default on a file case (no CUDA device needed; prints
//                                                                  its wall time as host_ms)
//          test_lookup_multiplicities random <k> <seed>           device == host default on random cases, and the same Panic text
// in.bin:  u32 k | u32 n_inputs | u64 usable | table (2^k x 32 B) | inputs (n_inputs x 2^k x 32 B), raw Montgomery limbs
// out.bin: u64 status (0 counted, 1 Panic) | m (2^k x 32 B) when counted
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <fstream>

#include "../../scroll-prover_b200/plonk_b200.hpp"

using namespace halo2_b200;
using namespace halo2_b200::plonk;

#define REQUIRE(c)                                                     \
    do {                                                               \
        if (!(c)) {                                                    \
            std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); \
            return 1;                                                  \
        }                                                              \
    } while (0)

// the Ops defaults alone: every other operation is out of this driver's scope
struct HostOps : Ops {
    [[noreturn]] static void no() { throw Panic("HostOps: not used here"); }
    G1 commit_lagrange(const Poly&) override { no(); }
    G1 commit(const Poly&) override { no(); }
    Poly lagrange_to_coeff(Poly) override { no(); }
    Poly coeff_to_extended(const Poly&) override { no(); }
    Poly extended_to_coeff(Poly) override { no(); }
    Fr eval_polynomial(const Poly&, const Fr&) override { no(); }
    Poly kate_division(const Poly&, const Fr&) override { no(); }
    Poly poly_mul(const Poly&, const Poly&) override { no(); }
    Poly poly_lincomb(const std::vector<const Poly*>&, const std::vector<Fr>&) override { no(); }
    void graph_evaluate(const Program&, const std::vector<const Poly*>&, const std::vector<const Poly*>&, const std::vector<const Poly*>&,
                        const std::vector<Fr>&, const Fr&, const Fr&, const Fr&, const Fr&, Poly&) override { no(); }
    Poly permutation_product(const std::vector<const Poly*>&, const std::vector<const Poly*>&, const Fr&, const Fr&, const Fr&, const Fr&,
                             const Fr&) override { no(); }
    Poly logup_running_sum(const std::vector<const Poly*>&, const Poly&, const Poly&, const Fr&, const Fr&) override { no(); }
};

// m, or the Panic text when the lookup is not satisfied
static std::pair<Poly, std::string> count(Ops& ops, const std::vector<Poly>& inputs, const Poly& table, uint64_t usable) {
    std::vector<const Poly*> in;
    for (auto& c : inputs) in.push_back(&c);
    try {
        return {ops.lookup_multiplicities(in, table, usable), ""};
    } catch (const Panic& e) {
        return {Poly(), e.what()};
    }
}

static int host_file(const char* in_path, const char* out_path) {
    std::ifstream f(in_path, std::ios::binary);
    uint32_t k = 0, n_inputs = 0;
    uint64_t usable = 0;
    f.read((char*)&k, 4).read((char*)&n_inputs, 4).read((char*)&usable, 8);
    const size_t n = size_t(1) << k;
    Poly table(n);
    std::vector<Poly> inputs(n_inputs, Poly(n));
    f.read((char*)table.data(), 32 * n);
    for (auto& c : inputs) f.read((char*)c.data(), 32 * n);
    REQUIRE(f.good());
    HostOps ops;
    const auto t0 = std::chrono::steady_clock::now();
    auto [m, panic] = count(ops, inputs, table, usable);
    std::printf("host_ms %.3f\n", std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    std::ofstream o(out_path, std::ios::binary);
    const uint64_t status = panic.empty() ? 0 : 1;
    o.write((const char*)&status, 8);
    if (panic.empty()) o.write((const char*)m.data(), 32 * n);
    else std::printf("panic: %s\n", panic.c_str());
    std::printf("OK\n");
    return 0;
}

static int random_cases(uint32_t k, uint64_t seed) {
    const uint64_t n = 1ull << k;
    EvaluationDomain dom = EvaluationDomain::new_(3, k);
    ParamsKZG params;
    DeviceOps dev(params, dom);
    HostOps host;
    Rng rng(seed);
    const uint64_t usable = n > 8 ? n - 7 : n;  // blinding rows at the end, as create_proof leaves them
    for (uint32_t n_inputs : {1u, 4u}) {
        // a table with duplicated values (a pool of n/4 distinct values) and inputs drawn from its usable rows
        std::vector<Fr> pool(std::max<uint64_t>(1, n / 4));
        for (auto& v : pool) v = rng.fr();
        Poly table(n);
        for (uint64_t r = 0; r < n; ++r) table[r] = r < usable ? pool[rng.next() % pool.size()] : rng.fr();  // rows >= usable: fresh values
        std::vector<Poly> inputs(n_inputs, Poly(n));
        for (auto& c : inputs)
            for (uint64_t r = 0; r < n; ++r) c[r] = (r < usable) ? table[rng.next() % usable] : rng.fr();
        auto [mh, ph] = count(host, inputs, table, usable);
        auto [md, pd] = count(dev, inputs, table, usable);
        REQUIRE(ph.empty() && pd.empty());
        REQUIRE(md == mh);
        // one input cell whose value is only in a row >= usable (or nowhere): both throw the same Panic
        const uint64_t bad = rng.next() % usable;
        inputs[n_inputs - 1][bad] = usable < n ? table[n - 1] : rng.fr();
        bool only_unusable = true;
        for (uint64_t r = 0; r < usable; ++r) only_unusable &= !(table[r] == inputs[n_inputs - 1][bad]);
        REQUIRE(only_unusable);
        auto [mh2, ph2] = count(host, inputs, table, usable);
        auto [md2, pd2] = count(dev, inputs, table, usable);
        REQUIRE(!ph2.empty() && ph2 == pd2);
        std::printf("k=%u inputs=%u: device m == host m; unsatisfied lookup -> \"%s\"\n", k, n_inputs, pd2.c_str());
    }
    std::printf("OK\n");
    return 0;
}

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    try {
        if (mode == "host" && argc > 3) return host_file(argv[2], argv[3]);
        if (mode == "random" && argc > 3) return random_cases((uint32_t)std::atoi(argv[2]), (uint64_t)std::atoll(argv[3]));
        std::printf("usage: %s host <in.bin> <out.bin> | random <k> <seed>\n", argv[0]);
        return 2;
    } catch (const std::exception& e) {
        std::printf("EXCEPTION: %s\n", e.what());
        return 1;
    }
}
