// eventgrad_b200 -- fused ring gossip step with gradient tracking (decent, --gradient-tracking), sm_90a.
// Same source as the default kernel, compiled with EG_GT: y, the previous gradient and the y inboxes travel in a
// separate TrackSlots block (api.h) that the launcher packs with GossipParams into the kernel's GtStepParams argument;
// GossipParams itself is unchanged (see the header comment of gossip.cu).  TrainConfig.gradient_tracking selects it.
#define EG_GT 1
#include "gossip.cu"
