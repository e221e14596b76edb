// create_proof with a proving key that holds no extended cosets: evaluate_h runs one coset part at a time
// (plonk_b200.hpp, keygen(..., keep_cosets = false)).  h(X) is unique, so the proof bytes must equal the whole-coset prover's.
// The circuits are those of test_plonk_session.cpp, included here unchanged.
//   usage: test_quotient_parts oracle|both|device [k] [seed] [variant]
//   oracle: over the CPU oracle (oracle_parts_ops.hpp): the by-parts proof (Blake2b transcript) is printed for the digest check
//           and must verify; with the Poseidon transcript it must equal the whole-coset oracle proof byte for byte
//   both:   additionally the by-parts prover through the C ABI (DeviceOps): identical bytes to the oracle's proof
//   device: the CUDA path alone at a larger size, Poseidon transcript: by parts == whole coset, both verifiers accept
#define main plonk_session_main
#include "test_plonk_session.cpp"
#undef main

#include "oracle_parts_ops.hpp"

int main(int argc, char** argv) {
    const std::string mode = argc > 1 ? argv[1] : "oracle";
    const uint32_t k = argc > 2 ? (uint32_t)std::atoi(argv[2]) : 6;
    const uint64_t seed = argc > 3 ? (uint64_t)std::atoll(argv[3]) : 1;
    const int variant = argc > 4 ? std::atoi(argv[4]) : 1;
    const uint64_t n = 1ull << k;
    try {
        Circuit C = variant == 3 ? build_phased(k, seed, 0) : (variant == 2 ? build_wide(k, seed, 0) : build(k, seed, 0));
        auto prove = [&](Ops& ops, const EvaluationDomain& dom, const ProvingKey& pk, uint64_t rng_seed, TranscriptKind kind) {
            return C.synth ? create_proof(ops, dom, pk, C.synth, C.instances, rng_seed, kind)
                           : create_proof(ops, dom, pk, C.advice, C.instances, rng_seed, kind);
        };
        EvaluationDomain dom = EvaluationDomain::new_(C.cs.degree(), k);
        const Fr tau = f_from_bytes_wide((const uint8_t*)"b200zk test srs: tau is NOT secret -- a toxic-waste-free toy..!!");
        VerifierParams vp;
        vp.g2 = pairing::g2_generator();
        {
            uint8_t repr[32];
            f_to_repr(tau, repr);
            uint64_t limbs[4];
            std::memcpy(limbs, repr, 32);
            vp.s_g2 = pairing::g2_mul(vp.g2, limbs);
        }
        std::string why;
        auto no_cosets = [](const ProvingKey& pk) {
            return pk.l0.empty() && pk.l_last.empty() && pk.l_active_row.empty() && pk.fixed_cosets.empty() && pk.sigma_cosets.empty() &&
                   !pk.l0_poly.empty() && !pk.l_last_poly.empty() && !pk.l_blind_poly.empty();
        };

        if (mode == "device") {
            ParamsKZG params;
            ParamsKZG::setup(params, k, tau);
            DeviceOps dops(params, dom);
            ProvingKey pk_w = keygen(dops, dom, C.cs, C.fixed, *C.assembly);
            ProvingKey pk_p = keygen(dops, dom, C.cs, C.fixed, *C.assembly, false);
            REQUIRE(no_cosets(pk_p) && pk_p.vk.transcript_repr == pk_w.vk.transcript_repr);
            ProofArtifacts pw = prove(dops, dom, pk_w, 0xB200 + seed, TranscriptKind::Poseidon);
            ProofArtifacts pp = prove(dops, dom, pk_p, 0xB200 + seed, TranscriptKind::Poseidon);
            REQUIRE(pp.proof == pw.proof);
            REQUIRE(verify_proof(dom, pk_p.vk, vp, C.instances, pp.proof, &why, TranscriptKind::Poseidon));
            protocol::PlonkProtocol P = protocol::parse_protocol(export_protocol_json(dom, pk_p.vk));
            const uint64_t u = n - C.cs.blinding_factors() - 1;
            std::vector<std::vector<Fr>> inst;
            for (auto& col : C.instances) inst.emplace_back(col.begin(), col.begin() + u);
            REQUIRE(snark::verify(P, inst, pp.proof, vp.g2, vp.s_g2, &why));
            std::printf("device proof of 2^%u rows by %u coset parts: %zu bytes, identical to the whole-coset proof, accepted by both verifiers\nOK\n",
                        k, dom.n_parts(), pp.proof.size());
            return 0;
        }

        std::vector<G1Affine> g(n), gl(n);
        halo2_params_setup(k, reinterpret_cast<const fr_t*>(&tau), reinterpret_cast<g1_affine_t*>(g.data()),
                           reinterpret_cast<g1_affine_t*>(gl.data()), 4);
        oracle_ops::OraclePartsOps oops(g, gl, C.cs.degree(), k);
        ProvingKey pk_p = keygen(oops, dom, C.cs, C.fixed, *C.assembly, false);
        REQUIRE(no_cosets(pk_p));
        ProofArtifacts po = prove(oops, dom, pk_p, 0xB200 + seed, TranscriptKind::Blake2b);
        std::printf("proof_sha_input parts_oracle %s\n", hex(po.proof).c_str());
        REQUIRE(verify_proof(dom, pk_p.vk, vp, C.instances, po.proof, &why));
        {   // the whole-coset oracle prover, Poseidon transcript: the same bytes
            ProvingKey pk_w = keygen(oops, dom, C.cs, C.fixed, *C.assembly);
            ProofArtifacts pw = prove(oops, dom, pk_w, 0xB200 + seed, TranscriptKind::Poseidon);
            ProofArtifacts pp = prove(oops, dom, pk_p, 0xB200 + seed, TranscriptKind::Poseidon);
            REQUIRE(pp.proof == pw.proof);
            REQUIRE(verify_proof(dom, pk_p.vk, vp, C.instances, pp.proof, &why, TranscriptKind::Poseidon));
            std::printf("poseidon proof by parts identical to the whole-coset one: %zu bytes\n", pp.proof.size());
        }
        if (mode == "both") {
            ParamsKZG params;
            params.k = k; params.n = n; params.g = g; params.g_lagrange = gl;
            DeviceOps dops(params, dom);
            ProvingKey pk_d = keygen(dops, dom, C.cs, C.fixed, *C.assembly, false);
            REQUIRE(no_cosets(pk_d) && pk_d.vk.transcript_repr == pk_p.vk.transcript_repr);
            ProofArtifacts pd = prove(dops, dom, pk_d, 0xB200 + seed, TranscriptKind::Blake2b);
            std::printf("proof_sha_input parts_device %s\n", hex(pd.proof).c_str());
            REQUIRE(pd.proof == po.proof);
            std::printf("device proof by parts identical to the oracle's: %zu bytes\n", pd.proof.size());
        }
        std::printf("OK\n");
        return 0;
    } catch (const std::exception& e) {
        std::printf("EXCEPTION: %s\n", e.what());
        return 1;
    }
}
