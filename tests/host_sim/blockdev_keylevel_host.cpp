// TEST HELPER (not product code): blockdev_host.cpp's host build of the device-side block logic plus its key-level part
// (blockdev_keylevel.inc).  Built as a library of its own; every other entry point is blockdev_host.cpp's.
#include "blockdev_host.cpp"
#include "blockdev_keylevel.inc"
