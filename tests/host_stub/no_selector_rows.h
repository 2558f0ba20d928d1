// Forced include for a build of kt_host.cc that must take the whole-upload path for throttle deletions and selector edits although
// the engine it is linked against (the product library) has kt_update_selector_rows: compiled with
// -Dkt_update_selector_rows=kt_update_selector_rows_absent, the host layer's reference names a symbol nothing defines, and this
// keeps that reference weak (null at run time).  tests/test_selector_rows_host.py uses such a build as the twin plugin.
#pragma weak kt_update_selector_rows_absent
