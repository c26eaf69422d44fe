# oracle/depth.mk -- builds oracle/liborc_depth.so: the depth oracle (orc_depth.c) linked with the oracle sources it
# builds on, with the flags of oracle/Makefile.  `make -C oracle -f depth.mk liborc_depth.so`
include Makefile
liborc_depth.so: $(SRCS) orc_depth.c orc_math.h orc_api.h orc_camera.h
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) orc_depth.c -lm
