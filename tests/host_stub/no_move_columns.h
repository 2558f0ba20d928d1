// Forced include for a build of kt_host.cc that must take the whole-upload path for placement rule 4 and hole compaction although
// the engine it is linked against (the product library) has kt_move_throttle_columns: compiled with
// -Dkt_move_throttle_columns=kt_move_throttle_columns_absent, the host layer's reference names a symbol nothing defines, and this
// keeps that reference weak (null at run time).  tests/test_move_columns_host.py uses such a build as the twin plugin.
#pragma weak kt_move_throttle_columns_absent
