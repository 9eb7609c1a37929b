// eventgrad_b200 -- fused gossip step on circulant graphs beyond the ring (decent/event), sm_90a.
// Same source as the default kernel, compiled with EG_GRAPH: the 2|O| inbox slots travel in a separate GraphSlots
// block (api.h) that the launcher packs with GossipParams into the kernel's GraphStepParams argument; GossipParams
// itself is unchanged (see the header comment of gossip.cu and parallel/topology.py).  TrainConfig.topology selects it.
#define EG_GRAPH 1
#include "gossip.cu"
