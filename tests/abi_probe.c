/* Compiled by tests/test_abi.py with the system C compiler against include/cosmo_b200.h and linked with
 * libcosmo_b200.so: prints the layout the C header really has (sizeof / offsetof of every field the ctypes
 * mirror declares) and exercises the entry points that need no GPU, from plain C. */
#include <stddef.h>
#include <stdio.h>
#include <string.h>

#include "cosmo_b200.h"

#define F(type, field) printf(#type "." #field " %zu\n", offsetof(type, field))

int main(void) {
  printf("sizeof.cosmo_b200_csc %zu\n", sizeof(cosmo_b200_csc));
  printf("sizeof.cosmo_b200_set %zu\n", sizeof(cosmo_b200_set));
  printf("sizeof.cosmo_b200_problem %zu\n", sizeof(cosmo_b200_problem));
  printf("sizeof.cosmo_b200_settings %zu\n", sizeof(cosmo_b200_settings));
  printf("sizeof.cosmo_b200_result %zu\n", sizeof(cosmo_b200_result));
  F(cosmo_b200_set, type); F(cosmo_b200_set, max_iter); F(cosmo_b200_set, dim); F(cosmo_b200_set, l);
  F(cosmo_b200_set, u); F(cosmo_b200_set, alpha); F(cosmo_b200_set, tol);
  F(cosmo_b200_problem, m); F(cosmo_b200_problem, P); F(cosmo_b200_problem, A); F(cosmo_b200_problem, q);
  F(cosmo_b200_problem, n_sets); F(cosmo_b200_problem, sets); F(cosmo_b200_problem, D); F(cosmo_b200_problem, c);
  F(cosmo_b200_settings, max_iter); F(cosmo_b200_settings, kkt_solver); F(cosmo_b200_settings, adaptive_rho_tolerance);
  F(cosmo_b200_settings, time_limit); F(cosmo_b200_settings, verbose); F(cosmo_b200_settings, psd_max_sweeps);
  F(cosmo_b200_settings, accelerator); F(cosmo_b200_settings, accelerator_mem); F(cosmo_b200_settings, accelerator_min_mem);
  F(cosmo_b200_settings, safeguard); F(cosmo_b200_settings, safeguard_tol);
  F(cosmo_b200_settings, adaptive_rho_fraction); F(cosmo_b200_settings, setup_time); F(cosmo_b200_settings, MAX_SCALING);
  F(cosmo_b200_settings, obj_true); F(cosmo_b200_settings, obj_true_tol);
  F(cosmo_b200_result, obj_val); F(cosmo_b200_result, iter); F(cosmo_b200_result, safeguarding_iter);
  F(cosmo_b200_result, status); F(cosmo_b200_result, r_prim); F(cosmo_b200_result, rho_updates);
  F(cosmo_b200_result, solver_time); F(cosmo_b200_result, kernel_launches);

  cosmo_b200_settings st;
  if (cosmo_b200_default_settings(&st) != COSMO_B200_OK) return 2;
  printf("abi %d\n", cosmo_b200_abi_version());
  printf("defaults %g %g %g %lld %d %d %g\n", st.rho, st.sigma, st.alpha, (long long)st.max_iter, st.accelerator,
         st.accelerator_mem, st.safeguard_tol);
  /* a null problem must be refused with an error code, not a crash */
  cosmo_b200_handle* h = NULL;
  int rc = cosmo_b200_create(&h, NULL, &st);
  printf("create_null %d\n", rc);
  const char* msg = cosmo_b200_last_error(NULL);
  printf("last_error %s\n", msg ? msg : "(null)");
  /* the test hooks refuse a null handle or null buffers the same way */
  double out8[8], lam = 0.0, v = 0.0;
  printf("infeasibility_null %d %d\n", cosmo_b200_infeasibility_test(NULL, 0, &v, out8),
         cosmo_b200_infeasibility_test(NULL, 0, NULL, NULL));
  printf("lambda_max_null %d %d\n", cosmo_b200_psd_lambda_max(NULL, &v, &lam), cosmo_b200_psd_lambda_max(NULL, NULL, &lam));
  return 0;
}
