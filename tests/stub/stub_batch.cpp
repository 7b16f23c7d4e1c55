// TEST INFRASTRUCTURE: the stand-in library of stub_aa.cpp plus kb_bus_set_batch_barcodes, so that the command line's
// handling of `bus --batch` with a technology and --batch-barcodes runs on a CPU-only box
// (tests/test_cli_bus_batch_host.py).  The stand-in's records carry the sample of kb_bus_begin_sample as their UMI;
// kb_bus_set_batch_barcodes says on stderr that it was called.  Never linked into the product.
#include <cstdio>

#include "stub_aa.cpp"

extern "C" {
int kb_bus_set_batch_barcodes(kb_quant*, int32_t on) { fprintf(stderr, "stub: batch barcodes %d\n", on); return KB_OK; }
}
