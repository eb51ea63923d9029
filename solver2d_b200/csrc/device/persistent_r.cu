// solver2d-b200 — the instantiation of the persistent kernel that runs the restitution pass (see persistent.cuh, solver.cu)
#include "persistent.cuh"

void* s2bRestitutionKernel()
{
	return (void*)s2bPersistentSolveT<S2B_RESTITUTION_PROGRAM>;
}
