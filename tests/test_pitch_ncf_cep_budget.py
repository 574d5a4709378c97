"""Register and spill budget of k_pitch_ncf and k_pitch_cep, compiled for sm_90a exactly as audioflux_b200/csrc/Makefile
compiles pitch_ncf_cep.cu (with -fmad=false), through the shared checker of tests/test_register_budgets.py.  Runs
wherever nvcc is present; no GPU needed."""
import test_register_budgets as RB

# CTAs of up to 1024 threads; the launcher sizes them for 2048 threads per SM (65 536 registers / 32)
BUDGET = RB.Budget("pitch_ncf_cep.cu", {"k_pitch_ncf": "k_pitch_ncf", "k_pitch_cep": "k_pitch_cep"}, 32, 0, 0,
                   ("-fmad=false",))


def test_pitch_ncf_cep_budget():
    RB.test_kernel_budget(BUDGET)
