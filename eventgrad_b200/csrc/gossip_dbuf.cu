// eventgrad_b200 -- EXPERIMENTAL double-buffered dense gossip step (decent), sm_90a.
// Same source as the default kernel, compiled with EG_DBUF: inbox slot = step & 1, no WAR ack
// (see the header comment of gossip.cu).  TrainConfig.double_buffer selects it.
#define EG_DBUF 1
#include "gossip.cu"
