// eventgrad_b200 -- fused ring gossip step with exact diffusion (decent, --exact-diffusion), sm_90a.
// Same source as the default kernel, compiled with EG_ED: psi, the previous optimizer output, travels in a separate
// EdSlots block (api.h) that the launcher packs with GossipParams into the kernel's EdStepParams argument; GossipParams
// itself is unchanged (see the header comment of gossip.cu).  TrainConfig.exact_diffusion selects it.
#define EG_ED 1
#include "gossip.cu"
