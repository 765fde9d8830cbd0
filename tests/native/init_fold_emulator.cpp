// init_fold_emulator.cpp -- host emulation of a schedule that starts from a pending basis state (test infrastructure).
//
// The schedule is planned like emul_schedule_jit (plan_emulator.cpp) does it, and every pass runs through its generated
// kernel compiled for the HOST (g++ -DQIP_JIT_HOST), except that the first pass is generated as a SYNTHESISED pass: its
// tiles are built from the basis index instead of being loaded.  The caller fills the state with garbage first, so any
// amplitude the synthesised pass reads instead of writing shows up in the result.
#include "plan_emulator.cpp"

// stats: [0] passes run through generated code, [1] single-op steps, [2] 1 when the first pass was synthesised,
//        [3] source bytes of the first pass, [4] whether its source carries QIP_SYNTH 1
extern "C" int emul_init_fold_jit(int prec, uint32_t n, uint64_t init_index, const qip_op *ops, size_t n_ops, void *state,
                                  uint32_t T, uint32_t L, const char *workdir, uint64_t *stats, char *errbuf, size_t errlen) {
  std::vector<FlatOp> flat(n_ops);
  for (size_t i = 0; i < n_ops; ++i) {
    std::string err;
    int st = compile_op(&ops[i], (qip_prec)prec, n, &flat[i], &err);
    if (st != QIPB200_OK) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "%s", err.c_str());
      return st;
    }
  }
  PlanConfig cfg = default_plan_config((qip_prec)prec, n);
  if (T) cfg.T = T;
  if (L) cfg.L = L;
  std::vector<PlanStep> steps;
  plan_passes(flat, n, (qip_prec)prec, cfg, &steps);
  if (steps.empty() || !steps[0].is_pass) {
    if (errbuf && errlen) snprintf(errbuf, errlen, "the schedule does not start with a tile pass");
    return -3;
  }
  const uint64_t N = 1ull << n;
  uint64_t st_[8] = {0};
  for (size_t s = 0; s < steps.size(); ++s) {
    if (!steps[s].is_pass) {
      std::vector<cd> psi(N);
      for (uint64_t i = 0; i < N; ++i)
        psi[i] = prec == QIP_F32 ? cd(((float *)state)[2 * i], ((float *)state)[2 * i + 1])
                                 : cd(((double *)state)[2 * i], ((double *)state)[2 * i + 1]);
      apply_single(flat[steps[s].op_index], n, psi);
      for (uint64_t i = 0; i < N; ++i) {
        if (prec == QIP_F32) {
          ((float *)state)[2 * i] = (float)psi[i].real();
          ((float *)state)[2 * i + 1] = (float)psi[i].imag();
        } else {
          ((double *)state)[2 * i] = psi[i].real();
          ((double *)state)[2 * i + 1] = psi[i].imag();
        }
      }
      ++st_[1];
      continue;
    }
    JitProgram prog;
    std::string why;
    if (!jit_generate(steps[s].pass, (qip_prec)prec, &prog, &why, false, s == 0 ? &init_index : nullptr)) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "generator declined pass %zu: %s", s, why.c_str());
      return -4;
    }
    if (s == 0) {
      st_[2] = prog.synthesised ? 1 : 0;
      st_[3] = prog.source.size();
      st_[4] = prog.source.find("#define QIP_SYNTH 1\n") != std::string::npos ? 1 : 0;
    }
    char base[512];
    snprintf(base, sizeof(base), "%s/initpass_%d_%zu", workdir, (int)getpid(), s);
    const std::string cu = std::string(base) + ".cpp", so = std::string(base) + ".so";
    FILE *f = fopen(cu.c_str(), "w");
    if (!f) return -5;
    fwrite(prog.source.data(), 1, prog.source.size(), f);
    fclose(f);
    if (s == 0 && getenv("INIT_FOLD_KEEP_SOURCE")) {  // for compiling the device side offline (nvcc)
      const std::string keep = std::string(getenv("INIT_FOLD_KEEP_SOURCE"));
      FILE *k = fopen(keep.c_str(), "w");
      if (k) {
        fwrite(prog.source.data(), 1, prog.source.size(), k);
        fclose(k);
      }
    }
    const std::string cmd = "/usr/bin/g++ -x c++ -std=c++17 -O1 -ffp-contract=off -DQIP_JIT_HOST -fPIC -shared -o " + so + " " + cu +
                            " 2> " + std::string(base) + ".log";
    if (system(cmd.c_str()) != 0) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "g++ failed on the generated source of pass %zu (see %s.log)", s, base);
      return -6;
    }
    void *h = dlopen(so.c_str(), RTLD_NOW | RTLD_LOCAL);
    if (!h) {
      if (errbuf && errlen) snprintf(errbuf, errlen, "dlopen: %s", dlerror());
      return -7;
    }
    typedef void (*Fn)(void *, const void *, unsigned);
    Fn fn = (Fn)dlsym(h, "qip_host_pass");
    if (!fn) return -8;
    fn(state, prog.params.data(), n);
    dlclose(h);
    unlink(so.c_str());
    ++st_[0];
  }
  if (stats) memcpy(stats, st_, sizeof(st_));
  return 0;
}
