// eventgrad_b200 -- fused gossip step on random pairwise matchings (decent, --topology random-match), sm_90a.
// Same source as the default kernel, compiled with EG_MATCH: the partner of each step comes from a seeded random perfect
// matching that every rank computes itself, and the single inbox, flag block and `done` word travel in a separate
// MatchSlots block (api.h) that the launcher packs with GossipParams into the kernel's MatchStepParams argument;
// GossipParams itself is unchanged (see the header comment of gossip.cu, parallel/topology.py and PROTOCOL.md 1.17).
#define EG_MATCH 1
#include "gossip.cu"
