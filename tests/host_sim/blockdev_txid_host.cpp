// TEST HELPER (not product code): blockdev_v13_host.cpp's host build of the device-side block logic with the committed tx-id set
// (blockdev_txid.inc).  Built as a library of its own.
#include "blockdev_host.cpp"
#include "blockdev_keylevel.inc"
#include "blockdev_v13.inc"
#include "blockdev_txid.inc"
