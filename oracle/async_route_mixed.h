// TEST INFRASTRUCTURE.  Included by oracle/transfer_ref.cpp in place of the reference's src/async/async_mpm.cpp when
// oracle/transfer_mixed_ref.cpp is built (REF_ASYNC_SOURCE names this file): the same source, included where it lies, with
// every MPM<dim>::substep() the scheduler calls sent to harness_substep_mixed, the patch point that routes pools of several
// particle types (transfer_mixed_ref.cpp).  transfer_ref.cpp has already opened AsyncMPM's private section and undoes
// that after this include.
namespace taichi {
void harness_substep_mixed(MPM<3> *m);
inline void harness_substep_mixed(MPM<2> *) {}
}  // namespace taichi
#undef substep
#define substep() res; ::taichi::harness_substep_mixed(this)
#include REF_ASYNC_ROUTED_SOURCE
