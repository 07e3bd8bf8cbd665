// Test-only harness of the exact sweep warm-ups the work planner marks (WorkPlan::warm_exact): the batch planner harness
// (plan_harness.cpp) with one more export, loaded by tests/test_plan_warm_exact.py.
#include "plan_harness.cpp"

PH_EXPORT void ph_warm_exact(const PhPlan* h, int32_t* out) { std::copy(h->plan.warm_exact.begin(), h->plan.warm_exact.end(), out); }
