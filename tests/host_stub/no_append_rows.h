// Forced include for a build of kt_host.cc that must take the whole-upload path for throttle creations although the engine it is
// linked against (the product library) has kt_append_throttle_rows: compiled with
// -Dkt_append_throttle_rows=kt_append_throttle_rows_absent, the host layer's reference names a symbol nothing defines, and this
// keeps that reference weak (null at run time).  tests/test_append_rows_host.py uses such a build as the twin plugin.
#pragma weak kt_append_throttle_rows_absent
