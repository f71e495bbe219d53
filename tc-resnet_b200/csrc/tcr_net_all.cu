// tcr_net_all.cu — single translation unit for the network kernels: the resident step kernel (tcr_resident.cu) reuses the
// device bodies of the per-layer kernels, so they must be visible to one compilation (no relocatable device code needed).  The
// listener (tcr_listener.cu) drives the per-layer forward with conv0 reading windows in place, so it is compiled here as well.
#include "tcr_net_fwd.cu"
#include "tcr_net_bwd.cu"
#include "tcr_optim.cu"
#include "tcr_resident.cu"
#include "tcr_listener.cu"
