// TEST INFRASTRUCTURE: OracleOps plus graph_evaluate_part on the oracle's interpreter (halo2_graph_evaluate), so that
// create_proof can run evaluate_h by coset parts over the CPU oracle.  The part transforms keep Ops' default bodies, i.e. the
// oracle's whole-coset coeff_to_extended / extended_to_coeff.  Never part of the product.
//
// The interpreter evaluates ExtendedX as zeta * omega^row.  On part j the point of row r is (zeta * w^r) * w_ext^j with
// w = w_ext^J, so the interpreter run over 2^k rows with omega = w and rot_scale = 1 evaluates the part once every ExtendedX
// operand is multiplied by the constant w_ext^j: rewrite_for_part prepends t = ExtendedX * c (c appended to the constants),
// replaces every ExtendedX operand by t and shifts every intermediate index by one (the Python twin is tests/part_programs.py).
#pragma once
#include "oracle_ops.hpp"

namespace oracle_ops {

inline Program rewrite_for_part(const Program& p, const Fr& factor) {
    auto uses_x = [](const b200zk_value_source& s) { return s.kind == B200ZK_SRC_EXTENDED_X; };
    bool any = false;
    for (auto& c : p.calcs) any |= uses_x(c.a) || uses_x(c.b);
    for (auto& s : p.parts) any |= uses_x(s);
    if (!any) return p;
    auto move = [&](b200zk_value_source s) {
        if (uses_x(s)) return b200zk_value_source{B200ZK_SRC_INTERMEDIATE, 0, 0};
        if (s.kind == B200ZK_SRC_INTERMEDIATE) s.index += 1;
        return s;
    };
    Program q;
    q.constants = p.constants;
    q.constants.push_back(factor);
    q.rotations = p.rotations;
    b200zk_calculation t{};
    t.op = B200ZK_CALC_MUL;
    t.a = b200zk_value_source{B200ZK_SRC_EXTENDED_X, 0, 0};
    t.b = b200zk_value_source{B200ZK_SRC_CONSTANT, (uint32_t)p.constants.size(), 0};
    q.calcs.push_back(t);
    for (auto c : p.calcs) {
        c.a = move(c.a);
        c.b = move(c.b);
        q.calcs.push_back(c);
    }
    for (auto& s : p.parts) q.parts.push_back(move(s));
    return q;
}

class OraclePartsOps : public OracleOps {
  public:
    OraclePartsOps(const std::vector<G1Affine>& g, const std::vector<G1Affine>& g_lagrange, uint32_t j, uint32_t k)
        : OracleOps(g, g_lagrange, j, k) {
        if (halo2_domain_new(&d_, j, k) != 0) throw Panic("halo2_domain_new failed");
    }
    void graph_evaluate_part(const Program& p, const std::vector<const Poly*>& fixed, const std::vector<const Poly*>& advice,
                             const std::vector<const Poly*>& instance, const std::vector<Fr>& challenges, const Fr& beta, const Fr& gamma,
                             const Fr& theta, const Fr& y, uint32_t part, Poly& values) override {
        auto tab = [](const std::vector<const Poly*>& v) {
            std::vector<const fr_t*> t;
            for (auto* c : v) t.push_back(fr(*c));
            return t;
        };
        auto tf = tab(fixed), ta = tab(advice), ti = tab(instance);
        fr_t factor = fr_ONE, w = d_.extended_omega;  // w_ext^part, w = w_ext^J
        for (uint32_t i = 0; i < part; ++i) fr_mul(&factor, &factor, &d_.extended_omega);
        for (uint32_t i = d_.k; i < d_.extended_k; ++i) fr_sqr(&w, &w);
        Fr f;
        std::memcpy(&f, &factor, sizeof f);
        const Program q = rewrite_for_part(p, f);
        int rc = halo2_graph_evaluate(reinterpret_cast<const halo2_calculation_t*>(q.calcs.data()), (uint32_t)q.calcs.size(),
                                      reinterpret_cast<const halo2_value_source_t*>(q.parts.data()), fr(q.constants), q.rotations.data(),
                                      (uint32_t)q.rotations.size(), tf.data(), ta.data(), ti.data(),
                                      reinterpret_cast<const fr_t*>(challenges.data()), fr1(beta), fr1(gamma), fr1(theta), fr1(y), &w,
                                      fr(values), d_.k, 1);
        if (rc != 0) throw Panic("halo2_graph_evaluate failed");
    }

  private:
    halo2_domain_t d_;
};
}  // namespace oracle_ops
