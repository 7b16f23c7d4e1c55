// TEST INFRASTRUCTURE: the stand-in library of stub_abi.cpp plus the `bus --aa` entry points, so that the command line's
// handling of --aa runs on a CPU-only box (tests/test_cli_aa_host.py).  kb_bus_set_aa accepts and changes nothing;
// kb_bus_frame_clashes reports the number of read sets the stand-in was given.  Never linked into the product.
#include "stub_abi.cpp"

extern "C" {
int kb_bus_set_aa(kb_quant*, int32_t) { return KB_OK; }
int kb_bus_frame_clashes(kb_quant* q, uint64_t* n) { *n = q->n; return KB_OK; }
}
