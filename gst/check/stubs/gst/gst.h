/* gst/check/stubs/gst/gst.h — DECLARATIONS ONLY, for `make -C gst/check` (gcc -fsyntax-only of the element sources in an
 * image without GLib / GStreamer).  Every prototype is restated from the reference headers named beside it
 * (/root/reference/subprojects/gstreamer/gst/ headers and GLib's public API); nothing here is ever linked.  Type checking
 * of the vmethod assignments is the point: the class structs carry the reference's vmethod signatures. */
#ifndef B200_STUB_GST_H
#define B200_STUB_GST_H
#include <stddef.h>
#include <stdint.h>
#include <string.h>

/* ---- GLib basics (glib/gtypes.h, gmacros.h) */
typedef int gint; typedef unsigned int guint; typedef int gboolean; typedef char gchar; typedef unsigned char guint8;
typedef size_t gsize; typedef int64_t gint64; typedef uint64_t guint64; typedef double gdouble; typedef float gfloat;
typedef void *gpointer; typedef const void *gconstpointer; typedef unsigned long gulong; typedef uint32_t guint32;
typedef gsize GType;
#define TRUE 1
#define FALSE 0
#define G_BEGIN_DECLS
#define G_END_DECLS
#define G_STMT_START do
#define G_STMT_END while (0)
#define G_MAXINT 2147483647
#define G_MININT (-2147483647 - 1)
#define G_MAXUINT 4294967295u
#define MIN(a, b) ((a) < (b) ? (a) : (b))
#define MAX(a, b) ((a) > (b) ? (a) : (b))
#define CLAMP(x, lo, hi) ((x) < (lo) ? (lo) : (x) > (hi) ? (hi) : (x))
#define G_N_ELEMENTS(a) (sizeof (a) / sizeof ((a)[0]))
typedef struct _GList { gpointer data; struct _GList *next, *prev; } GList;
gpointer g_malloc0 (gsize n_bytes);
void g_free (gpointer mem);
#define g_new0(T, n) ((T *) g_malloc0 (sizeof (T) * (n)))
#define g_clear_pointer(pp, destroy) G_STMT_START { if (*(pp)) { (destroy) (*(pp)); *(pp) = NULL; } } G_STMT_END
gboolean g_once_init_enter (void *location);
void g_once_init_leave (void *location, gsize result);

/* ---- GObject (gobject/gobject.h, gparam.h, gvalue.h, genums.h) */
typedef struct _GValue GValue; typedef struct _GParamSpec GParamSpec;
typedef struct _GTypeInstance { gpointer g_class; } GTypeInstance;
typedef struct _GObject { GTypeInstance g_type_instance; guint ref_count; gpointer qdata; } GObject;
typedef struct _GObjectClass {
  GType g_type;
  void (*set_property) (GObject * object, guint property_id, const GValue * value, GParamSpec * pspec);
  void (*get_property) (GObject * object, guint property_id, GValue * value, GParamSpec * pspec);
  void (*dispose) (GObject * object);
  void (*finalize) (GObject * object);
} GObjectClass;
typedef enum { G_PARAM_READABLE = 1, G_PARAM_WRITABLE = 2, G_PARAM_READWRITE = 3, G_PARAM_STATIC_STRINGS = 0xe0 } GParamFlags;
typedef struct { gint value; const gchar *value_name; const gchar *value_nick; } GEnumValue;
GType g_enum_register_static (const gchar * name, const GEnumValue * values);
void g_object_class_install_property (GObjectClass * oclass, guint property_id, GParamSpec * pspec);
GParamSpec *g_param_spec_int (const gchar * name, const gchar * nick, const gchar * blurb, gint minimum, gint maximum, gint default_value, GParamFlags flags);
GParamSpec *g_param_spec_uint (const gchar * name, const gchar * nick, const gchar * blurb, guint minimum, guint maximum, guint default_value, GParamFlags flags);
GParamSpec *g_param_spec_double (const gchar * name, const gchar * nick, const gchar * blurb, gdouble minimum, gdouble maximum, gdouble default_value, GParamFlags flags);
GParamSpec *g_param_spec_boolean (const gchar * name, const gchar * nick, const gchar * blurb, gboolean default_value, GParamFlags flags);
GParamSpec *g_param_spec_enum (const gchar * name, const gchar * nick, const gchar * blurb, GType enum_type, gint default_value, GParamFlags flags);
gint g_value_get_int (const GValue * value); void g_value_set_int (GValue * value, gint v);
guint g_value_get_uint (const GValue * value); void g_value_set_uint (GValue * value, guint v);
gdouble g_value_get_double (const GValue * value); void g_value_set_double (GValue * value, gdouble v);
gboolean g_value_get_boolean (const GValue * value); void g_value_set_boolean (GValue * value, gboolean v);
gint g_value_get_enum (const GValue * value); void g_value_set_enum (GValue * value, gint v);
void b200_stub_warn_invalid_property (GObject * o, guint id, GParamSpec * p);
#define G_OBJECT_WARN_INVALID_PROPERTY_ID(o, id, p) b200_stub_warn_invalid_property ((GObject *) (o), (id), (p))
#define G_OBJECT_CLASS(k) ((GObjectClass *) (k))
#define G_OBJECT(o) ((GObject *) (o))
#define G_TYPE_INT ((GType) 6 << 2)
/* G_DEFINE_TYPE (gobject/gtype.h): the parts the sources rely on - parent_class, get_type, the two init prototypes */
#define G_DEFINE_TYPE(TN, t_n, T_P)                                         \
  static void t_n##_class_init (TN##Class * klass);                         \
  static void t_n##_init (TN * self);                                       \
  static gpointer t_n##_parent_class = NULL;                                \
  GType t_n##_get_type (void) { (void) t_n##_class_init; (void) t_n##_init; (void) t_n##_parent_class; return (GType) (T_P); }

/* ---- GstObject / GstElement / caps / buffers (gst/gstobject.h, gstelement.h, gstcaps.h, gstbuffer.h, ...) */
typedef guint64 GstClockTime;
#define GST_CLOCK_TIME_NONE ((GstClockTime) -1)
#define GST_CLOCK_TIME_IS_VALID(t) (((GstClockTime) (t)) != GST_CLOCK_TIME_NONE)
#define GST_SECOND ((GstClockTime) 1000000000)
typedef struct _GstObject { GObject object; gint lock; gchar *name; } GstObject;
#define GST_OBJECT_LOCK(o) ((void) (o))
#define GST_OBJECT_UNLOCK(o) ((void) (o))
typedef struct _GstContext GstContext; typedef struct _GstCaps GstCaps; typedef struct _GstStructure GstStructure;
typedef struct _GstCapsFeatures GstCapsFeatures; typedef struct _GstQuery GstQuery; typedef struct _GstEvent GstEvent;
typedef struct _GstMemory GstMemory; typedef struct _GstBufferPool GstBufferPool; typedef struct _GstPlugin GstPlugin;
typedef struct _GstPad GstPad;
typedef struct _GstElement { GstObject object; GList *sinkpads, *srcpads; } GstElement;
typedef struct _GstElementClass {
  GObjectClass parent_class;
  void (*set_context) (GstElement * element, GstContext * context);     /* gstelement.h */
} GstElementClass;
#define GST_ELEMENT(o) ((GstElement *) (o))
#define GST_ELEMENT_CLASS(k) ((GstElementClass *) (k))
typedef enum { GST_PAD_UNKNOWN, GST_PAD_SRC, GST_PAD_SINK } GstPadDirection;
typedef enum { GST_PAD_ALWAYS, GST_PAD_SOMETIMES, GST_PAD_REQUEST } GstPadPresence;
typedef struct { const gchar *name_template; GstPadDirection direction; GstPadPresence presence; const gchar *static_caps; } GstStaticPadTemplate;
#define GST_STATIC_CAPS(s) (s)
#define GST_STATIC_PAD_TEMPLATE(n, d, p, c) { n, d, p, c }
typedef enum { GST_FLOW_OK = 0, GST_FLOW_NOT_NEGOTIATED = -4, GST_FLOW_ERROR = -5, GST_FLOW_CUSTOM_SUCCESS = 100 } GstFlowReturn;
typedef enum { GST_MAP_READ = 1, GST_MAP_WRITE = 2, GST_MAP_FLAG_LAST = 1 << 16 } GstMapFlags;
typedef struct { GstMemory *memory; GstMapFlags flags; guint8 *data; gsize size, maxsize; } GstMapInfo;
typedef struct _GstBuffer { gpointer mini_object; GstBufferPool *pool; GstClockTime pts, dts, duration; guint64 offset, offset_end; guint flags; } GstBuffer;
#define GST_BUFFER_PTS(b) ((b)->pts)
#define GST_BUFFER_DURATION(b) ((b)->duration)
#define GST_BUFFER_OFFSET(b) ((b)->offset)
#define GST_BUFFER_OFFSET_END(b) ((b)->offset_end)
enum { GST_BUFFER_FLAG_DISCONT = 1 << 6, GST_BUFFER_FLAG_GAP = 1 << 10 };
#define GST_BUFFER_FLAG_IS_SET(b, f) (((b)->flags & (f)) != 0)
#define GST_BUFFER_FLAG_SET(b, f) ((b)->flags |= (f))
#define GST_BUFFER_IS_DISCONT(b) GST_BUFFER_FLAG_IS_SET (b, GST_BUFFER_FLAG_DISCONT)
#define GST_MEMORY_FLAG_UNSET(m, f) ((void) (m))
gboolean gst_buffer_map (GstBuffer * buffer, GstMapInfo * info, GstMapFlags flags);
void gst_buffer_unmap (GstBuffer * buffer, GstMapInfo * info);
void gst_buffer_set_size (GstBuffer * buffer, gsize size);
GstMemory *gst_buffer_peek_memory (GstBuffer * buffer, guint idx);
GstBuffer *gst_buffer_new_and_alloc (gsize size);
void gst_buffer_unref (GstBuffer * buf);
GstFlowReturn gst_pad_push (GstPad * pad, GstBuffer * buffer);
typedef enum { GST_CAPS_INTERSECT_ZIG_ZAG, GST_CAPS_INTERSECT_FIRST } GstCapsIntersectMode;
GstCaps *gst_static_pad_template_get_caps (GstStaticPadTemplate * templ);
GstCaps *gst_caps_new_empty (void); GstCaps *gst_caps_copy (const GstCaps * caps); void gst_caps_unref (GstCaps * caps);
GstCaps *gst_caps_from_string (const gchar * string);   /* gstcaps.h:570 */
guint gst_caps_get_size (const GstCaps * caps); GstStructure *gst_caps_get_structure (const GstCaps * caps, guint index);
GstCapsFeatures *gst_caps_get_features (const GstCaps * caps, guint index);
gboolean gst_caps_features_contains (const GstCapsFeatures * features, const gchar * feature);
void gst_caps_append (GstCaps * caps1, GstCaps * caps2); void gst_caps_set_value (GstCaps * caps, const char *field, const GValue * value);
GstCaps *gst_caps_intersect_full (GstCaps * caps1, GstCaps * caps2, GstCapsIntersectMode mode);
GstCaps *gst_caps_truncate (GstCaps * caps); GstCaps *gst_caps_make_writable (GstCaps * caps); GstCaps *gst_caps_fixate (GstCaps * caps);
const GValue *gst_structure_get_value (const GstStructure * structure, const gchar * fieldname);
void gst_structure_set_value (GstStructure * structure, const gchar * fieldname, const GValue * value);
gboolean gst_structure_has_field (const GstStructure * structure, const gchar * fieldname);
const gchar *gst_structure_get_string (const GstStructure * structure, const gchar * fieldname);
gboolean gst_structure_get_int (const GstStructure * structure, const gchar * fieldname, gint * value);
gboolean gst_structure_fixate_field_nearest_int (GstStructure * structure, const char *field_name, int target);
gboolean gst_structure_fixate_field_string (GstStructure * structure, const char *field_name, const gchar * target);
void gst_structure_set (GstStructure * structure, const gchar * fieldname, ...);
#define GST_TYPE_INT_RANGE ((GType) 0x1234)
typedef enum { GST_QUERY_CONTEXT = 1, GST_QUERY_ALLOCATION = 2 } GstQueryType;
GstQueryType b200_stub_query_type (GstQuery * q);
#define GST_QUERY_TYPE(q) b200_stub_query_type (q)
typedef enum { GST_EVENT_FLUSH_STOP = 1, GST_EVENT_SEGMENT = 2, GST_EVENT_EOS = 3 } GstEventType;
GstEventType b200_stub_event_type (GstEvent * e);
#define GST_EVENT_TYPE(e) b200_stub_event_type (e)
void gst_query_parse_allocation (GstQuery * query, GstCaps ** caps, gboolean * need_pool);
guint gst_query_get_n_allocation_pools (GstQuery * query);
void gst_query_parse_nth_allocation_pool (GstQuery * query, guint index, GstBufferPool ** pool, guint * size, guint * min_buffers, guint * max_buffers);
void gst_query_set_nth_allocation_pool (GstQuery * query, guint index, GstBufferPool * pool, guint size, guint min_buffers, guint max_buffers);
void gst_query_add_allocation_pool (GstQuery * query, GstBufferPool * pool, guint size, guint min_buffers, guint max_buffers);
void gst_query_add_allocation_meta (GstQuery * query, GType api, const GstStructure * params);
GstStructure *gst_buffer_pool_get_config (GstBufferPool * pool);
gboolean gst_buffer_pool_set_config (GstBufferPool * pool, GstStructure * config);
void gst_buffer_pool_config_set_params (GstStructure * config, GstCaps * caps, guint size, guint min_buffers, guint max_buffers);
void gst_buffer_pool_config_add_option (GstStructure * config, const gchar * option);
void gst_object_unref (gpointer object);
#define gst_clear_object(pp) g_clear_pointer ((pp), gst_object_unref)
gboolean gst_util_fraction_multiply (gint a_n, gint a_d, gint b_n, gint b_d, gint * res_n, gint * res_d);
guint64 gst_util_uint64_scale_int (guint64 val, gint num, gint denom);
guint64 gst_util_uint64_scale_int_round (guint64 val, gint num, gint denom);
void gst_element_class_add_static_pad_template (GstElementClass * klass, GstStaticPadTemplate * static_templ);
void gst_element_class_add_static_pad_template_with_gtype (GstElementClass * klass, GstStaticPadTemplate * static_templ, GType pad_type);
void gst_element_class_set_static_metadata (GstElementClass * klass, const gchar * longname, const gchar * classification, const gchar * description, const gchar * author);
typedef enum { GST_RANK_NONE = 0 } GstRank;
gboolean gst_element_register (GstPlugin * plugin, const gchar * name, guint rank, GType type);
enum { GST_PARAM_CONTROLLABLE = 1 << 9, GST_PARAM_MUTABLE_READY = 1 << 10 };
/* debug / error macros (gst/gstinfo.h, gstelement.h) */
#define GST_DEBUG_CATEGORY_STATIC(c) static int c
#define GST_DEBUG_CATEGORY_INIT(c, name, color, desc) ((c) = 0)
void b200_stub_log (gpointer obj, const char *fmt, ...);
#define GST_ERROR_OBJECT(o, ...) b200_stub_log ((gpointer) (o), __VA_ARGS__)
#define GST_WARNING_OBJECT(o, ...) b200_stub_log ((gpointer) (o), __VA_ARGS__)
#define GST_DEBUG_OBJECT(o, ...) b200_stub_log ((gpointer) (o), __VA_ARGS__)
#define B200_STUB_UNPAREN(...) __VA_ARGS__
#define GST_ELEMENT_ERROR(el, domain, code, text, debug) G_STMT_START { b200_stub_log ((gpointer) (el), B200_STUB_UNPAREN text); b200_stub_log ((gpointer) (el), B200_STUB_UNPAREN debug); } G_STMT_END
#define GST_VERSION_MAJOR 1
#define GST_VERSION_MINOR 29
#define GST_PLUGIN_DEFINE(major, minor, name, description, init, version, license, package, origin) \
  gboolean b200_stub_plugin_entry_##name (GstPlugin * p) { return init (p); }
#endif
