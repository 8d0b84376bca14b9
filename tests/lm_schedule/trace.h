// Launch-schedule trace of lm_step.cu: shared by the CUDA-runtime stub (runtime.cpp), the generated launcher stubs and
// the driver.  Every pointer is printed as <buffer>+<byte offset> of a named buffer, so the trace does not depend on
// where the host allocator put anything.
#pragma once
#include <stddef.h>

// name a caller-owned buffer [base, base + bytes)
void tr_register(const char* name, const void* base, size_t bytes);
void tr_unregister(const void* base);
// "<name>+<offset>", "null", or "?" for an address outside every buffer
const char* tr_ptr(const void* p);
// one trace line (printf format, newline added)
void tr_log(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
