// mv_lookup::Argument::prepare's compression of the lookup input / table tuples with theta: Ops::compress_expressions, whose
// default body is the host fold over the expressions, against the programs keygen lowers for it (compression_program), run by
// the oracle's interpreter and by DeviceOps (b200zk_graph_evaluate with log_size = k, rot_scale = 1).  The session circuits are
// those of test_plonk_session.cpp, included here unchanged.
//   usage: test_lookup_compress host <in.bin> <out.bin>       the host default and the lowered programs of a file case (no device;
//                                                             prints its wall time as host_ms)
//          test_lookup_compress device <in.bin> <out.bin|->   DeviceOps == host default == oracle interpreter on a file case;
//                                                             writes the device columns unless out is "-"
//          test_lookup_compress session <k> <seed> <variant>  create_proof over the oracle with the compression done by the oracle's
//                                                             interpreter running the keygen programs, whole-coset and coset-free keys
//          test_lookup_compress session_device <k> <seed> <variant>   create_proof on the device, every compression checked
//                                                             against the host default element for element
//          test_lookup_compress tables                        column tables with unreferenced entries; a column index not supplied
//          test_lookup_compress time <in.bin> <reps>          DeviceOps: median of reps calls after two warm-ups; host default once
// in.bin:  u32 k | u32 n_fixed | u32 n_advice | u32 n_instance | u32 n_challenges | u32 n_sides | theta | challenges |
//          fixed, advice, instance columns (2^k elements each) | per side: u32 n_exprs, then each expression in prefix form:
//          u32 kind (Expr::Kind) | Constant: value | Fixed / Advice / Instance: u32 column, i32 rotation | Challenge: u32 index |
//          Negated: child | Sum, Product: child, child | Scaled: child, value          (field elements: 32 B, Montgomery limbs)
// out.bin: per side the 2^k compressed values; host mode then appends per side its program: u32 n_calcs | calcs (b200zk_calculation)
//          | u32 n_parts | parts (b200zk_value_source) | u32 n_constants | constants | u32 n_rotations | rotations (i32)
#include <algorithm>
#include <chrono>
#include <fstream>

#define main plonk_session_main
#include "test_plonk_session.cpp"
#undef main

#include "oracle_parts_ops.hpp"

namespace {

// the Ops defaults alone: every other operation is out of this driver's file modes
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

// the programs on the oracle's interpreter over the 2^k Lagrange rows (rotations wrap mod 2^k, as upstream's evaluate)
std::vector<Poly> oracle_compress(const std::vector<Program>& programs, const std::vector<Poly>& fixed, const std::vector<Poly>& advice,
                                  const std::vector<Poly>& instances, const std::vector<Fr>& challenges, const Fr& theta, uint32_t k) {
    using oracle_ops::OracleOps;
    auto tab = [](const std::vector<Poly>& v) {
        std::vector<const fr_t*> t;
        for (auto& c : v) t.push_back(OracleOps::fr(c));
        return t;
    };
    auto tf = tab(fixed), ta = tab(advice), ti = tab(instances);
    const Fr zero = f_zero();
    std::vector<Poly> out;
    for (const Program& p : programs) {
        Poly v((size_t)1 << k, f_zero());
        int rc = halo2_graph_evaluate(reinterpret_cast<const halo2_calculation_t*>(p.calcs.data()), (uint32_t)p.calcs.size(),
                                      reinterpret_cast<const halo2_value_source_t*>(p.parts.data()), OracleOps::fr(p.constants),
                                      p.rotations.data(), (uint32_t)p.rotations.size(), tf.data(), ta.data(), ti.data(),
                                      reinterpret_cast<const fr_t*>(challenges.data()), OracleOps::fr1(zero), OracleOps::fr1(zero),
                                      OracleOps::fr1(theta), OracleOps::fr1(zero), nullptr, OracleOps::fr(v), k, 1);
        if (rc != 0) throw Panic("halo2_graph_evaluate failed");
        out.push_back(std::move(v));
    }
    return out;
}

// OraclePartsOps whose compression is the oracle's interpreter running keygen's programs: create_proof's proof bytes then pin
// the program family to the host fold
struct CompressOracleOps : oracle_ops::OraclePartsOps {
    CompressOracleOps(const std::vector<G1Affine>& g, const std::vector<G1Affine>& gl, uint32_t j, uint32_t k)
        : OraclePartsOps(g, gl, j, k), k_(k) {}
    std::vector<Poly> compress_expressions(const std::vector<const std::vector<ExprP>*>& sides, const std::vector<Program>& programs,
                                           const std::vector<Poly>& fixed, const std::vector<Poly>& advice, const std::vector<Poly>& instances,
                                           const std::vector<Fr>& challenges, const Fr& theta) override {
        if (programs.size() != sides.size()) throw Panic("CompressOracleOps: one program per side");
        sides_run += programs.size();
        return oracle_compress(programs, fixed, advice, instances, challenges, theta, k_);
    }
    uint32_t k_;
    size_t sides_run = 0;
};

// DeviceOps whose every compression is also computed by the host default and must be identical
struct CheckedDeviceOps : DeviceOps {
    using DeviceOps::DeviceOps;
    std::vector<Poly> compress_expressions(const std::vector<const std::vector<ExprP>*>& sides, const std::vector<Program>& programs,
                                           const std::vector<Poly>& fixed, const std::vector<Poly>& advice, const std::vector<Poly>& instances,
                                           const std::vector<Fr>& challenges, const Fr& theta) override {
        auto dev = DeviceOps::compress_expressions(sides, programs, fixed, advice, instances, challenges, theta);
        auto host = Ops::compress_expressions(sides, programs, fixed, advice, instances, challenges, theta);
        if (dev != host) throw Panic("CheckedDeviceOps: device compression differs from the host default");
        sides_checked += sides.size();
        return dev;
    }
    size_t sides_checked = 0;
};

struct Case {
    uint32_t k = 0;
    Fr theta{};
    std::vector<Fr> challenges;
    std::vector<Poly> fixed, advice, instances;
    std::vector<std::vector<ExprP>> sides;
    std::vector<const std::vector<ExprP>*> side_ptrs() const {
        std::vector<const std::vector<ExprP>*> s;
        for (auto& x : sides) s.push_back(&x);
        return s;
    }
    std::vector<Program> programs() const {
        std::vector<Program> p;
        for (auto& x : sides) p.push_back(compression_program(x));
        return p;
    }
};

template <typename T>
T get(std::istream& f) {
    T v{};
    f.read((char*)&v, sizeof v);
    if (!f.good()) throw Panic("case file: truncated");
    return v;
}

ExprP read_expr(std::istream& f) {
    const uint32_t kind = get<uint32_t>(f);
    switch (kind) {
        case Expr::Constant: return Expr::constant(get<Fr>(f));
        case Expr::Fixed: { const uint32_t c = get<uint32_t>(f); return Expr::fixed(c, get<int32_t>(f)); }
        case Expr::Advice: { const uint32_t c = get<uint32_t>(f); return Expr::advice(c, get<int32_t>(f)); }
        case Expr::Instance: { const uint32_t c = get<uint32_t>(f); return Expr::instance(c, get<int32_t>(f)); }
        case Expr::Challenge: return Expr::challenge(get<uint32_t>(f));
        case Expr::Negated: return Expr::neg(read_expr(f));
        case Expr::Sum: { ExprP a = read_expr(f); return Expr::sum(a, read_expr(f)); }
        case Expr::Product: { ExprP a = read_expr(f); return Expr::mul(a, read_expr(f)); }
        case Expr::Scaled: { ExprP a = read_expr(f); return Expr::scaled(a, get<Fr>(f)); }
        default: throw Panic("case file: unknown expression kind");
    }
}

Case read_case(const char* path) {
    std::ifstream f(path, std::ios::binary);
    Case c;
    c.k = get<uint32_t>(f);
    const uint32_t nf = get<uint32_t>(f), na = get<uint32_t>(f), ni = get<uint32_t>(f), nc = get<uint32_t>(f), ns = get<uint32_t>(f);
    c.theta = get<Fr>(f);
    for (uint32_t i = 0; i < nc; ++i) c.challenges.push_back(get<Fr>(f));
    const size_t n = size_t(1) << c.k;
    for (auto [cols, cnt] : {std::make_pair(&c.fixed, nf), std::make_pair(&c.advice, na), std::make_pair(&c.instances, ni)})
        for (uint32_t i = 0; i < cnt; ++i) {
            cols->emplace_back(n);
            f.read((char*)cols->back().data(), 32 * n);
        }
    for (uint32_t s = 0; s < ns; ++s) {
        c.sides.emplace_back();
        const uint32_t m = get<uint32_t>(f);
        for (uint32_t e = 0; e < m; ++e) c.sides.back().push_back(read_expr(f));
    }
    if (!f.good()) throw Panic("case file: truncated");
    return c;
}

template <typename T>
void put_vec(std::ostream& o, const std::vector<T>& v) {
    const uint32_t n = (uint32_t)v.size();
    o.write((const char*)&n, 4);
    o.write((const char*)v.data(), sizeof(T) * v.size());
}

double ms_since(std::chrono::steady_clock::time_point t0) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

int host_file(const char* in_path, const char* out_path) {
    const Case c = read_case(in_path);
    const std::vector<Program> programs = c.programs();
    HostOps ops;
    const auto t0 = std::chrono::steady_clock::now();
    auto out = ops.compress_expressions(c.side_ptrs(), programs, c.fixed, c.advice, c.instances, c.challenges, c.theta);
    std::printf("host_ms %.3f\n", ms_since(t0));
    std::ofstream o(out_path, std::ios::binary);
    for (auto& col : out) o.write((const char*)col.data(), 32 * col.size());
    for (auto& p : programs) {
        put_vec(o, p.calcs);
        put_vec(o, p.parts);
        put_vec(o, p.constants);
        put_vec(o, p.rotations);
    }
    REQUIRE(o.good());
    std::printf("OK\n");
    return 0;
}

int device_file(const char* in_path, const char* out_path) {
    const Case c = read_case(in_path);
    const std::vector<Program> programs = c.programs();
    EvaluationDomain dom = EvaluationDomain::new_(3, c.k);
    ParamsKZG params;
    DeviceOps dev(params, dom);
    HostOps host;
    auto d = dev.compress_expressions(c.side_ptrs(), programs, c.fixed, c.advice, c.instances, c.challenges, c.theta);
    auto h = host.compress_expressions(c.side_ptrs(), programs, c.fixed, c.advice, c.instances, c.challenges, c.theta);
    auto o = oracle_compress(programs, c.fixed, c.advice, c.instances, c.challenges, c.theta, c.k);
    REQUIRE(d.size() == c.sides.size());
    REQUIRE(d == h);
    REQUIRE(d == o);
    if (std::string(out_path) != "-") {
        std::ofstream f(out_path, std::ios::binary);
        for (auto& col : d) f.write((const char*)col.data(), 32 * col.size());
        REQUIRE(f.good());
    }
    std::printf("k=%u sides=%zu: device == host default == oracle interpreter\nOK\n", c.k, d.size());
    return 0;
}

int time_file(const char* in_path, int reps) {
    const Case c = read_case(in_path);
    const std::vector<Program> programs = c.programs();
    EvaluationDomain dom = EvaluationDomain::new_(3, c.k);
    ParamsKZG params;
    DeviceOps dev(params, dom);
    HostOps host;
    auto& be = Backend::get();
    std::vector<Poly> d;
    for (int i = 0; i < 2; ++i) d = dev.compress_expressions(c.side_ptrs(), programs, c.fixed, c.advice, c.instances, c.challenges, c.theta);
    // the call ends with the download of every result column, a device synchronisation: the host clock around it is the
    // device-side time of the call, uploads included
    std::vector<double> ms;
    for (int i = 0; i < reps; ++i) {
        be.check(b200zk_ctx_synchronize(be.ctx()), "synchronize");
        const auto t0 = std::chrono::steady_clock::now();
        d = dev.compress_expressions(c.side_ptrs(), programs, c.fixed, c.advice, c.instances, c.challenges, c.theta);
        ms.push_back(ms_since(t0));
    }
    std::sort(ms.begin(), ms.end());
    std::printf("device_ms_median %.3f\ndevice_ms_min %.3f\n", ms[ms.size() / 2], ms.front());
    const auto t0 = std::chrono::steady_clock::now();
    auto h = host.compress_expressions(c.side_ptrs(), programs, c.fixed, c.advice, c.instances, c.challenges, c.theta);
    std::printf("host_ms %.3f\n", ms_since(t0));
    REQUIRE(d == h);
    std::printf("device == host default\nOK\n");
    return 0;
}

// create_proof over the CPU oracle with the compression on the oracle's interpreter: whole-coset and coset-free keys
int session(uint32_t k, uint64_t seed, int variant, bool on_device) {
    const uint64_t n = 1ull << k;
    Circuit C = variant == 3 ? build_phased(k, seed, 0) : (variant == 2 ? build_wide(k, seed, 0) : build(k, seed, 0));
    auto prove = [&](Ops& ops, const EvaluationDomain& dom, const ProvingKey& pk) {
        return C.synth ? create_proof(ops, dom, pk, C.synth, C.instances, 0xB200 + seed, TranscriptKind::Blake2b)
                       : create_proof(ops, dom, pk, C.advice, C.instances, 0xB200 + seed, TranscriptKind::Blake2b);
    };
    EvaluationDomain dom = EvaluationDomain::new_(C.cs.degree(), k);
    const Fr tau = f_from_bytes_wide((const uint8_t*)"b200zk test srs: tau is NOT secret -- a toxic-waste-free toy..!!");
    std::vector<G1Affine> g(n), gl(n);
    halo2_params_setup(k, reinterpret_cast<const fr_t*>(&tau), reinterpret_cast<g1_affine_t*>(g.data()),
                       reinterpret_cast<g1_affine_t*>(gl.data()), 4);
    const size_t n_sides = 2 * C.cs.lookups.size();
    if (on_device) {
        ParamsKZG params;
        params.k = k; params.n = n; params.g = g; params.g_lagrange = gl;
        CheckedDeviceOps dops(params, dom);
        for (bool keep_cosets : {true, false}) {
            ProvingKey pk = keygen(dops, dom, C.cs, C.fixed, *C.assembly, keep_cosets);
            REQUIRE(pk.lookup_compression.size() == n_sides);
            const size_t before = dops.sides_checked;
            ProofArtifacts pr = prove(dops, dom, pk);
            REQUIRE(dops.sides_checked == before + n_sides);
            std::printf("proof_sha_input %s %s\n", keep_cosets ? "device_whole" : "device_parts", hex(pr.proof).c_str());
        }
        std::printf("device compression == host default on %zu sides\nOK\n", dops.sides_checked);
        return 0;
    }
    CompressOracleOps oops(g, gl, C.cs.degree(), k);
    for (bool keep_cosets : {true, false}) {
        ProvingKey pk = keygen(oops, dom, C.cs, C.fixed, *C.assembly, keep_cosets);
        REQUIRE(pk.lookup_compression.size() == n_sides && pk.has_cosets() == keep_cosets);
        const size_t before = oops.sides_run;
        ProofArtifacts pr = prove(oops, dom, pk);
        REQUIRE(oops.sides_run == before + n_sides);
        std::printf("proof_sha_input %s %s\n", keep_cosets ? "whole" : "parts", hex(pr.proof).c_str());
    }
    std::printf("compression by the keygen programs on the oracle interpreter: %zu sides\nOK\n", oops.sides_run);
    return 0;
}

// Column tables: entries no program reads are never uploaded (here they are empty, which an upload would refuse), and a program
// reading a column beyond the supplied ones is refused by the ABI with its message
int tables() {
    const uint32_t k = 7;
    const size_t n = size_t(1) << k;
    Rng rng(42);
    auto col = [&]() {
        Poly p(n);
        for (auto& v : p) v = rng.fr();
        return p;
    };
    Case c;
    c.k = k;
    c.theta = rng.fr();
    c.challenges = {rng.fr(), rng.fr()};
    c.fixed = {Poly(), Poly(), col(), Poly(), Poly(), col()};
    c.advice = {Poly(), col(), Poly(), col()};
    c.instances = {Poly(), col()};
    c.sides = {{Expr::mul(Expr::fixed(5), Expr::advice(1, -1)), Expr::advice(3, 2)},
               {Expr::fixed(2)},
               {Expr::sum(Expr::instance(1), Expr::challenge(1)), Expr::mul(Expr::fixed(5), Expr::advice(3))}};
    EvaluationDomain dom = EvaluationDomain::new_(3, k);
    ParamsKZG params;
    DeviceOps dev(params, dom);
    HostOps host;
    const auto programs = c.programs();
    auto d = dev.compress_expressions(c.side_ptrs(), programs, c.fixed, c.advice, c.instances, c.challenges, c.theta);
    auto h = host.compress_expressions(c.side_ptrs(), programs, c.fixed, c.advice, c.instances, c.challenges, c.theta);
    REQUIRE(d == h);
    std::printf("unreferenced entries: device == host default on %zu sides\n", d.size());
    c.sides.push_back({Expr::fixed(6)});  // one past the six supplied fixed columns
    std::string why;
    try {
        dev.compress_expressions(c.side_ptrs(), c.programs(), c.fixed, c.advice, c.instances, c.challenges, c.theta);
    } catch (const Panic& e) {
        why = e.what();
    }
    REQUIRE(!why.empty());
    std::printf("column not supplied -> %s\nOK\n", why.c_str());
    return 0;
}

}  // namespace

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "";
    try {
        if (mode == "host" && argc > 3) return host_file(argv[2], argv[3]);
        if (mode == "device" && argc > 3) return device_file(argv[2], argv[3]);
        if (mode == "time" && argc > 3) return time_file(argv[2], std::atoi(argv[3]));
        if ((mode == "session" || mode == "session_device") && argc > 4)
            return session((uint32_t)std::atoi(argv[2]), (uint64_t)std::atoll(argv[3]), std::atoi(argv[4]), mode == "session_device");
        if (mode == "tables") return tables();
        std::printf("usage: %s host <in> <out> | device <in> <out|-> | time <in> <reps> | session[_device] <k> <seed> <variant> | tables\n",
                    argv[0]);
        return 2;
    } catch (const std::exception& e) {
        std::printf("EXCEPTION: %s\n", e.what());
        return 1;
    }
}
