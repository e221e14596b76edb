// dev::MockProver::verify_par on the device: mock_prove(DeviceOps, ...) -- Ops::check_constraints over b200zk_nonzero_rows,
// b200zk_lookup_missing_rows and b200zk_copy_check -- against the host mock_prove (mock_check), element for element.  The session
// circuits are those of test_plonk_session.cpp, included here unchanged.
//   usage: test_mock_device host <k> <seed> <variant> <out.bin>   no device: the host mock_prove of the honest witness and sabotages
//                                                                1-4, with the inputs of the three checks, for tests/mock_model.py
//          test_mock_device device <k> <seed> <variant>           DeviceOps == host on the honest witness and sabotages 1-4
//          test_mock_device synthetic <k> <seed> <plants>         a circuit of 32 gates, 4 lookups into a 2^16 range table and 8
//                                                                permutation columns with random cycles, `plants` witness cells
//                                                                broken: DeviceOps == host
//          test_mock_device time <k> <seed> <plants> <reps>       the same circuit: DeviceOps median of reps calls after one warm-up,
//                                                                host once; the two lists are compared
// out.bin, per case (honest, then sabotage 1-4): u32 k | u64 usable | u32 n_gates | u32 n_lookups | u32 n_perm | each gate's values
//          (2^k Fr) | per lookup its compressed input, then table (2^k Fr each) | the permutation columns (2^k Fr each) | next
//          (n_perm * 2^k u64, c * 2^k + r) | u64 n_failures | per failure u32 kind, u32 index, u64 row      (Fr: Montgomery limbs)
#include <algorithm>
#include <chrono>
#include <fstream>

#define main plonk_session_main
#include "test_plonk_session.cpp"
#undef main

namespace {

// the Ops defaults alone: every other operation is out of this driver's host mode
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

WitnessFn witness_of(const Circuit& X) {
    if (X.synth) return X.synth;
    const std::vector<Poly>* adv = &X.advice;
    return [adv](uint32_t, const std::vector<Fr>&, std::vector<Poly>& table) { table = *adv; };
}

Circuit session_circuit(uint32_t k, uint64_t seed, int variant, int sabotage) {
    return variant == 3 ? build_phased(k, seed, sabotage) : (variant == 2 ? build_wide(k, seed, sabotage) : build(k, seed, sabotage));
}

const char* kind_name(int kind) { return kind == MockFailure::Gate ? "gate" : (kind == MockFailure::Lookup ? "lookup" : "permutation"); }

std::string summary(const std::vector<MockFailure>& f) {
    size_t c[3] = {0, 0, 0};
    for (auto& x : f) c[x.kind]++;
    return "gate " + std::to_string(c[0]) + ", lookup " + std::to_string(c[1]) + ", permutation " + std::to_string(c[2]);
}

// the first position where two failure lists differ, for the message of a mismatch
std::string first_difference(const std::vector<MockFailure>& a, const std::vector<MockFailure>& b) {
    size_t i = 0;
    while (i < a.size() && i < b.size() && a[i] == b[i]) ++i;
    auto show = [](const std::vector<MockFailure>& v, size_t i) {
        return i < v.size() ? std::string(kind_name(v[i].kind)) + " " + std::to_string(v[i].index) + " row " + std::to_string(v[i].row) : "end";
    };
    return "at " + std::to_string(i) + ": device " + show(a, i) + ", host " + show(b, i);
}

int host_dump(uint32_t k, uint64_t seed, int variant, const char* out_path) {
    const uint64_t n = 1ull << k;
    std::ofstream o(out_path, std::ios::binary);
    auto put = [&](const void* p, size_t bytes) { o.write((const char*)p, bytes); };
    HostOps ops;
    for (int sabotage = 0; sabotage <= 4; ++sabotage) {
        Circuit C = session_circuit(k, seed, variant, sabotage);
        EvaluationDomain dom = EvaluationDomain::new_(C.cs.degree(), k);
        const std::vector<MockFailure> f = mock_prove(dom, C.cs, C.fixed, *C.assembly, witness_of(C), C.instances, 7 + seed);
        const MockWitness w = mock_synthesize(dom, C.cs, C.fixed, witness_of(C), C.instances, 7 + seed);
        REQUIRE(ops.check_constraints(w.cs, C.fixed, w.advice, C.instances, w.challenges, w.theta, *C.assembly) == f);
        // the inputs of the three checks: each gate and lookup tuple evaluated by the host fold (Horner(0, [e], theta) = e)
        std::vector<std::vector<ExprP>> sides;
        for (auto& g : w.cs.gates) sides.push_back({g});
        for (auto& l : w.cs.lookups) { sides.push_back(l.inputs); sides.push_back(l.table); }
        std::vector<const std::vector<ExprP>*> sp;
        for (auto& s : sides) sp.push_back(&s);
        const std::vector<Poly> vals = ops.compress_expressions(sp, std::vector<Program>(sides.size()), C.fixed, w.advice, C.instances,
                                                                w.challenges, w.theta);
        const uint64_t u = n - w.cs.blinding_factors() - 1;
        put(&k, 4);
        put(&u, 8);
        const uint32_t counts[3] = {(uint32_t)w.cs.gates.size(), (uint32_t)w.cs.lookups.size(), (uint32_t)w.cs.permutation.size()};
        put(counts, 12);
        for (auto& v : vals) put(v.data(), 32 * n);
        for (const Column& c : w.cs.permutation) {
            const Poly& col = c.kind == Expr::Fixed ? C.fixed[c.index] : (c.kind == Expr::Advice ? w.advice[c.index] : C.instances[c.index]);
            put(col.data(), 32 * n);
        }
        std::vector<uint64_t> next;
        for (size_t c = 0; c < w.cs.permutation.size(); ++c)
            for (uint64_t r = 0; r < n; ++r) next.push_back((uint64_t)C.assembly->mapping[c][r].first * n + C.assembly->mapping[c][r].second);
        put(next.data(), 8 * next.size());
        const uint64_t nf = f.size();
        put(&nf, 8);
        for (auto& x : f) {
            const uint32_t ki[2] = {(uint32_t)x.kind, (uint32_t)x.index};
            put(ki, 8);
            put(&x.row, 8);
        }
        std::printf("sabotage %d: %zu failures (%s)\n", sabotage, f.size(), summary(f).c_str());
    }
    REQUIRE(o.good());
    std::printf("OK\n");
    return 0;
}

int device_session(uint32_t k, uint64_t seed, int variant) {
    for (int sabotage = 0; sabotage <= 4; ++sabotage) {
        Circuit C = session_circuit(k, seed, variant, sabotage);
        EvaluationDomain dom = EvaluationDomain::new_(C.cs.degree(), k);
        ParamsKZG params;
        DeviceOps dev(params, dom);
        const auto d = mock_prove(dev, dom, C.cs, C.fixed, *C.assembly, witness_of(C), C.instances, 7 + seed);
        const auto h = mock_prove(dom, C.cs, C.fixed, *C.assembly, witness_of(C), C.instances, 7 + seed);
        if (d != h) std::printf("mismatch %s\n", first_difference(d, h).c_str());
        REQUIRE(d == h);
        REQUIRE((sabotage == 0) == d.empty());
        std::printf("sabotage %d: device == host, %zu failures (%s)\n", sabotage, d.size(), summary(d).c_str());
    }
    std::printf("OK\n");
    return 0;
}

uint64_t mix(uint64_t x) {  // splitmix64
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// A circuit at the scale of the reference's MockProver runs.  Every advice column c holds w_c * x(row) with x a pseudo-random
// value below 2^16 (w = 1, 2, 3, 4, 5, 6, 1, 2), so that
//   32 gates  q_s * (w_j a_i - w_i a_j), the same at rotation 1, and q_s * (w_l w_m a_i a_j - w_i w_j a_l a_m), s = g mod 4
//   4 lookups q_l a_0 in T;  (q_l a_0, q_l a_1) in (T, 2T);  q_l a_2 in 3T;  q_l a_0(omega X) in T   (T = row mod 2^16)
//   copies    within each of the permutation columns a_0 .. a_5 between rows of equal x, and between a_0, a_6 and a_1, a_7 on a row
// all hold on the usable rows; the selectors are off from row u - 1 on (a rotation by 1 would read a blinding row).  Then
// `plants` random advice cells below u get + 1.
Circuit build_synthetic(uint32_t k, uint64_t seed, uint32_t plants) {
    Circuit C;
    const uint64_t n = 1ull << k;
    ConstraintSystem& cs = C.cs;
    const uint32_t A = 8, W[A] = {1, 2, 3, 4, 5, 6, 1, 2};
    cs.num_fixed = 6;  // q_0 .. q_3, q_l, T
    cs.num_advice = A;
    cs.num_instance = 0;
    auto a = [](uint32_t c, int32_t rot = 0) { return Expr::advice(c, rot); };
    auto sc = [](ExprP e, uint64_t v) { return Expr::scaled(e, f_u64(v)); };
    for (uint32_t g = 0; g < 32; ++g) {
        const uint32_t i = g % A, j = (g + 3) % A, l = (g + 2) % A, m = (g + 5) % A;
        const ExprP q = Expr::fixed(g % 4);
        if (g % 3 == 0) cs.gates.push_back(Expr::mul(q, Expr::sub(sc(a(i), W[j]), sc(a(j), W[i]))));
        if (g % 3 == 1) cs.gates.push_back(Expr::mul(q, Expr::sub(sc(a(i, 1), W[j]), sc(a(j, 1), W[i]))));
        if (g % 3 == 2)
            cs.gates.push_back(Expr::mul(q, Expr::sub(sc(Expr::mul(a(i), a((g + 1) % A)), W[l] * W[m]),
                                                      sc(Expr::mul(a(l), a(m)), W[i] * W[(g + 1) % A]))));
    }
    const ExprP ql = Expr::fixed(4), T = Expr::fixed(5);
    cs.lookups.push_back(Lookup{{Expr::mul(ql, a(0))}, {T}});
    cs.lookups.push_back(Lookup{{Expr::mul(ql, a(0)), Expr::mul(ql, a(1))}, {T, sc(T, 2)}});
    cs.lookups.push_back(Lookup{{Expr::mul(ql, a(2))}, {sc(T, 3)}});
    cs.lookups.push_back(Lookup{{Expr::mul(ql, a(0, 1))}, {T}});
    for (uint32_t c = 0; c < A; ++c) cs.permutation.push_back({Expr::Advice, c});
    cs.finalize();
    const uint64_t u = n - cs.blinding_factors() - 1;
    const uint64_t M = std::min<uint64_t>(1ull << 16, u - 8);  // x stays a usable row of T
    C.fixed.assign(6, Poly(n, f_zero()));
    C.advice.assign(A, Poly(n, f_zero()));
    C.instances.clear();
    std::vector<uint64_t> x(n, 0);
    for (uint64_t r = 0; r < u; ++r) x[r] = mix(seed * 0x1000003 + r) % M;
    for (uint64_t r = 0; r < n; ++r) {
        for (uint32_t s = 0; s < 4; ++s) C.fixed[s][r] = (r + 1 < u && (r + s) % 5 != 0) ? f_one() : f_zero();
        C.fixed[4][r] = (r + 1 < u && r % 3 != 0) ? f_one() : f_zero();
        C.fixed[5][r] = f_u64(r % (1ull << 16));
        for (uint32_t c = 0; c < A; ++c) C.advice[c][r] = f_u64(W[c] * x[r]);
    }
    C.assembly = std::make_unique<Assembly>(A, n);
    std::vector<uint64_t> by_x(u);
    for (uint64_t r = 0; r < u; ++r) by_x[r] = r;
    std::sort(by_x.begin(), by_x.end(), [&](uint64_t p, uint64_t q) { return x[p] != x[q] ? x[p] < x[q] : p < q; });
    uint64_t rng = mix(seed);
    for (uint32_t c = 0; c < 6; ++c)
        for (uint64_t t = 1; t < u; ++t) {
            rng = mix(rng);
            if (x[by_x[t]] == x[by_x[t - 1]] && rng % 3 == 0) C.assembly->copy(c, (uint32_t)by_x[t - 1], c, (uint32_t)by_x[t]);
        }
    for (uint64_t r = 0; r < u; ++r) {
        rng = mix(rng);
        if (rng % 4 == 0) C.assembly->copy(0, (uint32_t)r, 6, (uint32_t)r);
        if (rng % 4 == 1) C.assembly->copy(1, (uint32_t)r, 7, (uint32_t)r);
    }
    for (uint32_t p = 0; p < plants; ++p) {
        rng = mix(rng);
        const uint32_t c = (uint32_t)(rng % A);
        rng = mix(rng);
        const uint64_t r = rng % u;
        C.advice[c][r] = f_add(C.advice[c][r], f_one());
    }
    return C;
}

double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

int synthetic(uint32_t k, uint64_t seed, uint32_t plants, int reps) {
    Circuit C = build_synthetic(k, seed, plants);
    EvaluationDomain dom = EvaluationDomain::new_(C.cs.degree(), k);
    ParamsKZG params;
    DeviceOps dev(params, dom);
    const WitnessFn wit = witness_of(C);
    std::vector<MockFailure> d = mock_prove(dev, dom, C.cs, C.fixed, *C.assembly, wit, C.instances, seed);
    if (reps > 0) {
        // every call ends with the download of its failure counts and lists, a device synchronisation: the host clock around it is
        // the call's time, uploads included
        auto& be = Backend::get();
        std::vector<double> ms;
        for (int i = 0; i < reps; ++i) {
            be.check(b200zk_ctx_synchronize(be.ctx()), "synchronize");
            const auto t0 = std::chrono::steady_clock::now();
            d = mock_prove(dev, dom, C.cs, C.fixed, *C.assembly, wit, C.instances, seed);
            ms.push_back(ms_since(t0));
        }
        std::sort(ms.begin(), ms.end());
        std::printf("device_ms_median %.3f\ndevice_ms_min %.3f\n", ms[ms.size() / 2], ms.front());
    }
    const auto t0 = std::chrono::steady_clock::now();
    const std::vector<MockFailure> h = mock_prove(dom, C.cs, C.fixed, *C.assembly, wit, C.instances, seed);
    std::printf("host_ms %.3f\n", ms_since(t0));
    if (d != h) std::printf("mismatch %s\n", first_difference(d, h).c_str());
    REQUIRE(d == h);
    const uint64_t bf = C.cs.blinding_factors();
    std::printf("k=%u gates=%zu lookups=%zu permutation=%zu blinding=%llu: device == host, %zu failures (%s)\nOK\n", k, C.cs.gates.size(),
                C.cs.lookups.size(), C.cs.permutation.size(), (unsigned long long)bf, d.size(), summary(d).c_str());
    return 0;
}

}  // namespace

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    auto arg = [&](int i) { return (uint64_t)std::atoll(argv[i]); };
    try {
        if (mode == "host" && argc > 5) return host_dump((uint32_t)arg(2), arg(3), (int)arg(4), argv[5]);
        if (mode == "device" && argc > 4) return device_session((uint32_t)arg(2), arg(3), (int)arg(4));
        if (mode == "synthetic" && argc > 4) return synthetic((uint32_t)arg(2), arg(3), (uint32_t)arg(4), 0);
        if (mode == "time" && argc > 5) return synthetic((uint32_t)arg(2), arg(3), (uint32_t)arg(4), (int)arg(5));
        std::printf("usage: %s host <k> <seed> <variant> <out> | device <k> <seed> <variant> | synthetic <k> <seed> <plants> | "
                    "time <k> <seed> <plants> <reps>\n", argv[0]);
        return 2;
    } catch (const std::exception& e) {
        std::printf("EXCEPTION: %s\n", e.what());
        return 1;
    }
}
