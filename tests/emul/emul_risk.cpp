// TEST-ONLY: the ensemble risk measure of csrc/dial_device.cuh (ens_risk_derive on the host,
// ens_risk_reduce in the reduction kernel) compiled by g++ with -ffp-contract=off, so that the _rn
// intrinsic shims of the emulator build round each operation as the GPU does.  Built into its own library
// by tests/test_ensemble_risk.py.  Never loaded by the dial_mpc_b200 package.
#define DIAL_HOST_EMUL 1
#include "../../dial_mpc_b200/csrc/dial_device.cuh"

// The setting dial_plan_set_ensemble_risk derives: out = {mode, n_tail} and {frac, denom}.
extern "C" void emul_risk_derive(int K, int mode, float alpha, int32_t* iout, float* fout) {
  const EnsRisk R = ens_risk_derive(K, mode, alpha);
  iout[0] = R.mode; iout[1] = R.n_tail; fout[0] = R.frac; fout[1] = R.denom;
}

// The reduction kernel's per-sample work on member rewards r [K][n] (member k of sample i at k n + i).
extern "C" void emul_risk_reduce(const float* r, int K, int n, int mode, float alpha, float* out) {
  const EnsRisk R = ens_risk_derive(K, mode, alpha);
  for (int i = 0; i < n; ++i) out[i] = ens_risk_reduce(r + i, (size_t)n, K, R);
}
