// Step functions of the stand-alone L2 entry points (l12.cu): each runs the body of one entry point on device-resident arrays
// inside the caller's Stage, so that a batched driver (gg20_general.cu) composes them on its own scratch.  The entry points are
// these steps plus staging, and launch the same kernels in the same order.  `n` is the instance count of the step.
#pragma once
#include "stage.cuh"

namespace tecdsa {
int secp_mul_step(tecdsa_ctx* c, int n, const uint32_t* pts, const uint32_t* scalars, uint32_t* out);
int hash_commitment_step(tecdsa_ctx* c, int n, const uint32_t* points, const uint32_t* blind, uint32_t* com);
int pedersen_prove_step(tecdsa_ctx* c, int n, const uint32_t* m, const uint32_t* r, const uint32_t* s1, const uint32_t* s2, uint32_t* com, uint32_t* proof);
int pedersen_verify_step(tecdsa_ctx* c, int n, const uint32_t* com, const uint32_t* proof, uint8_t* status);
int heg_prove_step(tecdsa_ctx* c, int n, const uint32_t* G, const uint32_t* D, const uint32_t* E, const uint32_t* x, const uint32_t* r, const uint32_t* s1,
                   const uint32_t* s2, uint32_t* proof);
int heg_verify_step(tecdsa_ctx* c, int n, const uint32_t* G, const uint32_t* D, const uint32_t* E, const uint32_t* proof, uint8_t* status);
int alice_generate_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* sr, const uint32_t* da,
                        const uint32_t* dc, const uint32_t* dr, const uint32_t* dal, const uint32_t* dbe, const uint32_t* dga, const uint32_t* dro,
                        uint32_t* dz, uint32_t* de, uint32_t* ds, uint32_t* ds1, uint32_t* ds2);
int alice_verify_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* sr, const uint32_t* dc,
                      const uint32_t* dz, const uint32_t* de, const uint32_t* ds, const uint32_t* ds1, const uint32_t* ds2, uint8_t* dst);
int pdl_prove_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* sr, const uint32_t* dx, const uint32_t* dr,
                   const uint32_t* dc, const uint32_t* dQ, const uint32_t* dG, const uint32_t* dal, const uint32_t* dbe, const uint32_t* dro,
                   const uint32_t* dga, uint32_t* dz, uint32_t* du1, uint32_t* du2, uint32_t* du3, uint32_t* ds1, uint32_t* ds2, uint32_t* ds3);
int pdl_verify_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* sr, const uint32_t* dc, const uint32_t* dQ,
                    const uint32_t* dG, const uint32_t* dz, const uint32_t* du1, const uint32_t* du2, const uint32_t* du3, const uint32_t* ds1,
                    const uint32_t* ds2, const uint32_t* ds3, uint8_t* dst);
int mta_encrypt_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* da, const uint32_t* dr, uint32_t* dc);
int mta_message_a_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, int n_st, const uint32_t* er, const uint32_t* da, const uint32_t* dr,
                       const uint32_t* sr, const uint32_t* dal, const uint32_t* dbe, const uint32_t* dga, const uint32_t* dro, uint32_t* dc, uint32_t* dz,
                       uint32_t* de, uint32_t* ds, uint32_t* ds1, uint32_t* ds2);
int mta_message_b_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* er, const uint32_t* db, const uint32_t* dca, const uint32_t* dr,
                       const uint32_t* dbt, const uint32_t* dnb, const uint32_t* dnt, int n_st, const uint32_t* sr, const uint32_t* dz, const uint32_t* de,
                       const uint32_t* ds, const uint32_t* ds1, const uint32_t* ds2, const uint8_t* checked, uint32_t* dcb, uint32_t* dbp, uint32_t* dtp,
                       uint32_t* dbeta, uint8_t* dst);
int mta_get_alpha_step(tecdsa_ctx* c, Stage& S, const tecdsa_keyset* ks, int n, const uint32_t* dr, const uint32_t* da, const uint32_t* dcb, const uint32_t* dbp,
                       const uint32_t* dtp, uint32_t* dal, uint32_t* dpl, uint8_t* dst);
}  // namespace tecdsa
