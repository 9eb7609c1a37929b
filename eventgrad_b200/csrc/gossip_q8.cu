// eventgrad_b200 -- fused ring gossip step with int8 error-feedback compression of the pushes (decent/event), sm_90a.
// Same source as the default kernel, compiled with EG_Q8: the int8 code / scale inboxes, `prev` and the two neighbour
// replicas travel in a separate Q8Slots block (api.h) that the launcher packs with GossipParams into the kernel's
// Q8StepParams argument; GossipParams itself is unchanged (see the header comment of gossip.cu).  TrainConfig.compress
// selects it.
#define EG_Q8 1
#include "gossip.cu"
