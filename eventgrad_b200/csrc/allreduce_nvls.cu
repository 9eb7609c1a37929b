// eventgrad_b200 -- EXPERIMENTAL NVLink-SHARP (NVLS) all-reduce + 1/R + SGD, sm_90a.
// Same source as the default kernel, compiled with EG_NVLS: the owner of a tile reduces it inside the
// NVSwitch (multimem.ld_reduce on the multicast mapping) and broadcasts the average with multimem.st.
// Needs the window to live in torch symmetric memory (parallel/window.py:SymmWindow, EGB_NVLS=1).
#define EG_NVLS 1
#include "allreduce.cu"
